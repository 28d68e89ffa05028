"""ctypes binding of oracle/filtered_range_search.cpp (liboracle_filtered_range_search.so, oracle/filtered_range_search.mk,
built by build()), and an independent Python restatement of the reference's filtered range search to pin it.
TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as O
from range_oracle import check, deleted_words  # noqa: F401  (Range::validate_and_create's checks are the same)

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        O.lib()  # liboracle.so, which this library links against
        path = os.path.join(O.ORACLE_DIR, "liboracle_filtered_range_search.so")
        src = os.path.join(O.ORACLE_DIR, "filtered_range_search.cpp")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", O.ORACLE_DIR, "-s", "-f", "filtered_range_search.mk"], stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        vp, u32, u64, i, f = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_float
        L.orc_filtered_range_search.restype = u64
        L.orc_filtered_range_search.argtypes = [C.POINTER(O.OrcIndex), vp, u32, u32, f, i, f, f, f, u64, vp, u64, i, vp, i, vp, vp, vp, vp,
                                                vp]
        _LIB = L
    return _LIB


def range_search(index, queries, l_search, radius, labels, masks, match_all=False, beam=1, inner_radius=None, initial_slack=1.0,
                 range_slack=1.0, max_returned=None, deleted=None, flavour=O.AVX2):
    """orc_filtered_range_search over an O.Index, one query after another: (offsets [nq + 1] u64, ids, dists, cmps, hops,
    second_round) as range_oracle.range_search.  `labels`: u64 per id; `masks`: u64 per query (or one)."""
    assert check(l_search, radius, beam, inner_radius, initial_slack, range_slack, max_returned) is None
    queries = np.ascontiguousarray(queries)
    total = index.n_points + index.n_start
    labels = np.ascontiguousarray(labels, np.uint64)
    assert labels.shape == (total,)
    nq = queries.shape[0]
    masks = np.broadcast_to(np.asarray(masks, np.uint64), (nq,))
    words = None if deleted is None else deleted_words(deleted, total)
    ids = np.empty(max(index.n_points, 1), np.uint32)
    dists = np.empty(max(index.n_points, 1), np.float32)
    cmps, hops, second = np.empty(nq, np.uint32), np.empty(nq, np.uint32), np.empty(nq, np.uint8)
    offsets, all_ids, all_dists = [0], [], []
    c, h, s = C.c_uint32(), C.c_uint32(), C.c_uint8()
    for q in range(nq):
        n = lib().orc_filtered_range_search(C.byref(index.c), queries[q].ctypes.data, l_search, beam, radius, inner_radius is not None,
                                            0.0 if inner_radius is None else inner_radius, initial_slack, range_slack, max_returned or 0,
                                            O.ptr(labels), int(masks[q]), int(bool(match_all)), None if words is None else O.ptr(words),
                                            flavour, O.ptr(ids), O.ptr(dists), C.byref(c), C.byref(h), C.byref(s))
        all_ids.append(ids[:n].copy())
        all_dists.append(dists[:n].copy())
        offsets.append(offsets[-1] + n)
        cmps[q], hops[q], second[q] = c.value, h.value, s.value
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.empty(0, dt)
    return np.array(offsets, np.uint64), cat(all_ids, np.uint32), cat(all_dists, np.float32), cmps, hops, second


# ---------------------------------------------------------------- the reference's search, restated in Python

class Queue:
    """NeighborPriorityQueue::{insert, closest_notvisited} (queue.rs:130-171, 297-313)"""

    def __init__(self, cap):
        self.cap, self.items, self.cursor = cap, [], 0  # items: [distance, id, visited]

    def insert(self, i, d):
        if np.isnan(d) or (len(self.items) == self.cap and self.items[-1][0] < d):
            return
        at = next((j for j, x in enumerate(self.items) if x[0] >= d), len(self.items))
        if len(self.items) == self.cap:
            self.items.pop()
        self.items.insert(at, [d, i, False])
        self.cursor = min(self.cursor, at)

    def closest_notvisited(self):
        if self.cursor >= min(self.cap, len(self.items)):
            return None
        c = self.cursor
        self.items[c][2] = True
        self.cursor += 1
        while self.cursor < len(self.items) and self.items[self.cursor][2]:
            self.cursor += 1
        return self.items[c][1]


def py_search(vecs, adj, n_points, n_start, metric, query, L, radius, labels, mask, match_all=False, beam=1, inner_radius=None,
              initial_slack=1.0, range_slack=1.0, max_returned=None, deleted=None):
    """FilteredRange::search: (ids, dists, cmps, hops, second_round) of one query"""
    total = n_points + n_start
    limit = max_returned or float("inf")
    q = np.ascontiguousarray(query.astype(np.float32) if vecs.dtype == np.float16 else query)
    dist = lambda ids: O.distance_rows(q, vecs[np.asarray(ids, np.int64)], metric, O.AVX2) if len(ids) else []
    accept = lambda i: (int(labels[i]) & mask) == mask if match_all else (int(labels[i]) & mask) != 0
    radius, bound = np.float32(radius), np.float32(radius) * np.float32(range_slack)

    def expand(nodes, visited):
        fresh = []
        for u in nodes:
            for v in adj[u, 1:1 + adj[u, 0]].tolist():
                if v not in visited:
                    visited.add(v)
                    if v < total:
                        fresh.append(v)
        return fresh

    best, matched, visited = Queue(L + n_start), [], set(range(n_points, total))
    for i, d in zip(range(n_points, total), dist(list(range(n_points, total)))):
        best.insert(i, d)
        if accept(i):
            matched.append((i, d))
    cmps = hops = 0
    while True:
        nodes = []
        while len(nodes) < beam and (u := best.closest_notvisited()) is not None:
            nodes.append(u)
        if not nodes:
            break
        fresh = expand(nodes, visited)
        for i, d in zip(fresh, dist(fresh)):
            if accept(i):
                matched.append((i, d))
            best.insert(i, d)
        cmps += len(fresh)
        hops += len(nodes)
    matched.sort(key=lambda m: (bool(np.isnan(m[1])), 0.0 if np.isnan(m[1]) else float(m[1])))  # stable
    within = [m for m in matched if m[1] <= radius]
    in_range = sorted({(float(d), i) for d, i, _ in best.items[:L] if d <= radius} | {(float(d), i) for i, d in within})
    in_range = [i for _, i in in_range]  # (distance, id) order; an id has one distance, so the set removed its repeats
    second = len(in_range) >= int(np.float32(L) * np.float32(initial_slack)) and len(within) < limit
    if second:
        visited, frontier = set(in_range), list(in_range)
        head = 0
        while head < len(frontier) and len(within) < limit:
            nodes = frontier[head:head + beam]
            head += len(nodes)
            fresh = expand(nodes, visited)
            for i, d in zip(fresh, dist(fresh)):
                if d <= bound:
                    frontier.append(i)
                    if d <= radius and accept(i) and len(within) < limit:
                        within.append((i, d))
            cmps += len(fresh)
            hops += len(nodes)
    out = [(i, d) for i, d in within[:int(min(len(within), limit))]
           if not (inner_radius is not None and d <= inner_radius) and i < n_points and not (deleted is not None and deleted[i])]
    return (np.array([i for i, _ in out], np.uint32), np.array([d for _, d in out], np.float32), cmps, hops, bool(second))
