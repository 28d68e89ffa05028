"""Host-side model of the batched rank-merge the search kernels use (search_common.cuh,
merge_round) against the reference's sequential NeighborPriorityQueue::insert
(queue.rs:130-171, restated in oracle/graph.cpp): inserting a round of candidates one by one at
the lower bound, with tail eviction, must equal "keep the `cap` smallest under (distance
ascending, later-inserted first among equal distances)" computed by rank."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O


def sequential(cap, rounds):
    L = O.lib()
    q = L.orc_queue_new(cap)
    try:
        for ids, dists in rounds:
            for i, d in zip(ids, dists):
                L.orc_queue_insert(q, int(i), float(d))
        n = min(cap, L.orc_queue_size(q))
        out = []
        for k in range(n):
            i, d, v = C.c_uint32(), C.c_float(), C.c_int()
            L.orc_queue_get(q, k, C.byref(i), C.byref(d), C.byref(v))
            out.append((i.value, np.float32(d.value)))
        return out
    finally:
        L.orc_queue_free(q)


def merge_round(cap, old, ids, dists):
    """merge_round of search_common.cuh in numpy: `old` is the sorted list [(id, dist)]."""
    od = np.array([d for _, d in old], np.float32)
    size = len(old)
    worst = od[cap - 1] if size == cap else np.float32(np.inf)
    dists = np.asarray(dists, np.float32)
    valid = ~np.isnan(dists) & ~(worst < dists)        # NaN ignored; a full list pre-rejects worst < x
    new = [(int(i), np.float32(d), j) for j, (i, d) in enumerate(zip(ids, dists)) if valid[j]]
    out = {}
    for idn, d, j in new:
        lo = int(np.sum(od < d))                                                # lower bound among the old entries
        rn = sum(1 for _, e, k in new if e < d or (e == d and k > j))             # new entries ranked ahead: later first among ties
        pos = lo + rn
        if pos < cap:
            out[pos] = (idn, d)
    for e, (ido, d) in enumerate(old):
        sh = sum(1 for _, x, _ in new if x <= d)                                # an old entry moves right past every new x <= d
        if e + sh < cap:
            assert e + sh not in out
            out[e + sh] = (ido, np.float32(d))
    n = min(cap, size + len(new))
    assert sorted(out) == list(range(n)), "ranks must tile the list without holes"
    return [out[k] for k in range(n)]


@pytest.mark.parametrize("seed", range(12))
def test_rank_merge_equals_sequential_inserts(seed):
    rng = np.random.default_rng(seed)
    cap = int(rng.integers(1, 40))
    rounds, model, next_id = [], [], 0
    for _ in range(int(rng.integers(1, 9))):
        m = int(rng.integers(0, 33))                                             # a round is at most one warp of candidates
        # few distinct values -> many exact ties; sprinkle NaN and infinities
        d = rng.choice(np.array([0.0, 0.5, 1.0, 1.0, 2.0, 3.5, np.inf, np.nan, -1.0], np.float32), m).astype(np.float32)
        ids = np.arange(next_id, next_id + m, dtype=np.uint32)
        next_id += m
        rounds.append((ids, d))
        model = merge_round(cap, model, ids, d)
        want = sequential(cap, rounds)
        assert [(i, float(x)) for i, x in model] == [(i, float(x)) for i, x in want], (seed, cap, len(rounds))


def test_full_list_accepts_equal_to_worst_and_evicts_it():
    # queue.rs:141-143: only `last < new` is rejected; an equal distance enters before its equals
    old = [(1, np.float32(1.0)), (2, np.float32(2.0))]
    got = merge_round(2, old, np.array([7], np.uint32), np.array([2.0], np.float32))
    assert got == [(1, np.float32(1.0)), (7, np.float32(2.0))]
    assert got == sequential(2, [(np.array([1, 2]), np.array([1.0, 2.0])), (np.array([7]), np.array([2.0]))])


def merge_round_in_place_by_tiles(cap, old, ids, dists, tile):
    """merge_round_chunked of search_common.cuh: the list lives in one array and is rewritten IN PLACE, a tile of
    `tile` entries at a time from the top tile down (each tile: read all of it, then write the moved entries)."""
    size = len(old)
    qd = np.full(cap + 64, np.float32(np.nan), np.float32)
    qi = np.full(cap + 64, 0xFFFFFFFF, np.uint32)
    for e, (i, d) in enumerate(old):
        qi[e], qd[e] = i, d
    worst = qd[cap - 1] if size == cap else np.float32(np.inf)
    dists = np.asarray(dists, np.float32)
    valid = ~np.isnan(dists) & ~(worst < dists)
    new = [(int(i), np.float32(d), j) for j, (i, d) in enumerate(zip(ids, dists)) if valid[j]]
    if not new:
        return list(old)
    od_all = qd[:size].copy()
    placed = []
    for idn, d, j in new:
        pos = int(np.sum(od_all < d)) + sum(1 for _, e, k in new if e < d or (e == d and k > j))
        if pos < cap:
            placed.append((pos, idn, d))
    for c in range((size + tile - 1) // tile - 1, -1, -1):                         # from the top occupied tile down
        e0 = c * tile
        regs = [(e, qi[e], qd[e]) for e in range(e0, min(e0 + tile, size))]      # the whole tile is read first ...
        for e, i, d in regs:                                                    # ... then its moved entries are written
            sh = sum(1 for _, x, _ in new if x <= d)
            if sh != 0 and e + sh < cap:
                qi[e + sh], qd[e + sh] = i, d
    for pos, idn, d in placed:
        qi[pos], qd[pos] = idn, d
    n = min(cap, size + len(new))
    return [(int(qi[k]), np.float32(qd[k])) for k in range(n)]


@pytest.mark.parametrize("seed", range(16))
def test_tile_wise_in_place_merge_equals_the_rank_merge(seed):
    """Lists longer than one register tile (the PQ traversal with L > 512, search_kernel_v2 with L + start points > 256):
    walking the tiles from the top one down and rewriting the list in place gives the list the one-tile merge (and
    hence the sequential inserts) gives."""
    rng = np.random.default_rng(100 + seed)
    cap = int(rng.integers(5, 60))
    tile = int(rng.integers(2, 9))
    model, next_id = [], 0
    for _ in range(int(rng.integers(2, 10))):
        m = int(rng.integers(0, 33))
        d = rng.choice(np.array([0.0, 0.5, 1.0, 1.0, 2.0, 3.5, 7.0, np.inf, np.nan, -1.0], np.float32), m).astype(np.float32)
        ids = np.arange(next_id, next_id + m, dtype=np.uint32)
        next_id += m
        want = merge_round(cap, model, ids, d)
        got = merge_round_in_place_by_tiles(cap, model, ids, d, tile)
        assert [(i, float(x)) for i, x in got] == [(i, float(x)) for i, x in want], (seed, cap, tile)
        model = want
