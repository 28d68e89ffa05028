#!/usr/bin/env python3
"""How many f32 L2 search candidates a bound from the high 16 bits of their rows would reject.

    python tools/skip_fraction.py [--workload c2_1Mx128_f32_l2] [--queries 320] [--out DIR]

Builds the workload's graph on the device exactly as bench.py does, downloads it, and replays `--queries` queries of
bench.py's first batch on the host at the workload's L, with the oracle's queue semantics (capacity L + #start, a full
list rejects a candidate whose distance is above its last one) and the oracle's distances.  Every candidate of a round
that starts with a full list and a finite last distance `thr` is also given a lower bound: each element x is known only
to lie between the floats whose high 16 bits are those of x (low bits all 0 or all 1), and the bound sums, per element,
the squared distance from the query element to that interval (0 inside it).  A candidate counts as skipped when
bound * (1 - 2^-16) > thr.  The replay's cmps and hops are checked against the oracle's own search.

Reports the skipped fraction of all candidates and the candidate-row bytes per query: a whole row for every candidate
today, and with split rows half a row for every candidate plus the other half for every candidate not skipped.
Needs a GPU (the build); writes skip_fraction.json under --out.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def interval_bounds(rows):
    """Per element, the two floats whose high 16 bits are those of the row element (low bits 0 and 0xFFFF), ordered."""
    bits = np.ascontiguousarray(rows, np.float32).view(np.uint32) & np.uint32(0xFFFF0000)
    a = bits.view(np.float32)
    b = (bits | np.uint32(0xFFFF)).view(np.float32)
    finite = np.isfinite(a).all(1)
    return np.minimum(a, b), np.maximum(a, b), finite


def lower_bounds(q, rows):
    lo, hi, finite = interval_bounds(rows)
    q = q.astype(np.float64)[None, :]
    gap = np.maximum(lo.astype(np.float64) - q, 0.0) + np.maximum(q - hi.astype(np.float64), 0.0)
    return (gap * gap).sum(1), finite


def replay(q, vecs, adj, n_points, n_start, l_search, O):
    """Greedy search (beam 1) of one query; returns cmps, hops, candidates seen with a full list, skipped."""
    cap = l_search + n_start
    ids, dists, vis = [], [], []
    cursor = 0
    visited = set()

    def insert(i, d):
        nonlocal cursor
        if np.isnan(d):
            return
        if len(ids) == cap and dists[-1] < d:
            return
        idx = next((k for k, v in enumerate(dists) if v >= d), len(dists))
        if len(ids) == cap:
            ids.pop(), dists.pop(), vis.pop()
        ids.insert(idx, i), dists.insert(idx, d), vis.insert(idx, False)
        cursor = min(cursor, idx)

    total = n_points + n_start
    starts = list(range(n_points, total))
    sd = O.distance_rows(q, vecs[starts], O.L2, O.AVX2)
    for i, d in zip(starts, sd):
        visited.add(i)
        insert(i, float(d))
    cmps, hops, full_cands, skipped = len(starts), 0, 0, 0
    while cursor < min(cap, len(ids)):
        node = ids[cursor]
        vis[cursor] = True
        cursor += 1
        while cursor < len(ids) and vis[cursor]:
            cursor += 1
        hops += 1
        row = adj[node]
        cand = []
        for n in row[1:1 + row[0]]:
            n = int(n)
            if n in visited:
                continue
            visited.add(n)
            if n < total:
                cand.append(n)
        if not cand:
            continue
        d = O.distance_rows(q, vecs[cand], O.L2, O.AVX2)
        if len(ids) == cap and np.isfinite(dists[-1]):
            thr = dists[-1]
            lb, finite = lower_bounds(q, vecs[cand])
            skip = finite & (lb * (1.0 - 2.0 ** -16) > thr) & (np.asarray(cand) < n_points)
            assert not (skip & (d <= thr)).any(), "the bound rejected a candidate the list accepts"
            full_cands += len(cand)
            skipped += int(skip.sum())
        for i, v in zip(cand, d):
            insert(i, float(v))
        cmps += len(cand)
    return cmps, hops, full_cands, skipped


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workload", default="c2_1Mx128_f32_l2")
    ap.add_argument("--queries", type=int, default=320)
    ap.add_argument("--out", default=".", help="directory for skip_fraction.json")
    args = ap.parse_args()

    import bench
    import diskann_b200 as dab
    import oracle_lib as O

    cfg = bench.WORKLOADS[args.workload]
    assert cfg["dtype"] == "f32" and cfg["metric"] == "l2" and cfg["path"] == "fp", "f32 L2 full-precision workloads only"
    n, dim, md = cfg["n"], cfg["dim"], bench.max_degree(cfg["R"])
    t0 = time.time()
    centers = bench.make_centers(cfg)
    base = bench.make_data(cfg, bench.SEED_BASE, n, centers)
    medoid = bench.find_medoid(base)
    queries = bench.make_data(cfg, bench.SEED_QUERY, cfg["nq"], centers)[:args.queries]
    with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, dim, n, 1, md) as g:
        g.upload_vectors(base)
        g.upload_vectors(medoid[None, :], first=n)
        g.build(cfg["R"], cfg["l_build"], bench.ALPHA)
        adj = g.download_graph()
    t_build = time.time() - t0
    vecs = np.concatenate([base, medoid[None, :]])
    del base

    t0 = time.time()
    L = cfg["l_search"]
    oidx = O.Index(vecs, adj, n, 1, O.L2)
    _, _, _, want_cmps, want_hops = oidx.search_batch(queries, bench.K, L)
    cmps = np.zeros(len(queries), np.int64)
    hops = np.zeros(len(queries), np.int64)
    full = np.zeros(len(queries), np.int64)
    skipped = np.zeros(len(queries), np.int64)
    for i, q in enumerate(queries):
        cmps[i], hops[i], full[i], skipped[i] = replay(q, vecs, adj, n, 1, L, O)
    assert np.array_equal(cmps, want_cmps) and np.array_equal(hops, want_hops), "the replay left the oracle's search"
    row = dim * 4
    res = {
        "workload": args.workload, "queries": len(queries), "l_search": L,
        "cmps_per_query": float(cmps.mean()), "hops_per_query": float(hops.mean()),
        "candidates_with_full_list_fraction": float(full.sum() / cmps.sum()),
        "skipped_fraction": float(skipped.sum() / cmps.sum()),
        "skipped_fraction_per_query": {"min": float((skipped / cmps).min()), "median": float(np.median(skipped / cmps)),
                                       "max": float((skipped / cmps).max())},
        "row_bytes_per_query_today": float(cmps.mean() * row),
        "row_bytes_per_query_split": float(cmps.mean() * row / 2 + (cmps - skipped).mean() * row / 2),
        "build_s": round(t_build, 1), "replay_s": round(time.time() - t0, 1),
    }
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "skip_fraction.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
