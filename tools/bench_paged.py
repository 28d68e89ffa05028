"""Paged search on the C2 workload of bench.py, against the one-shot searches it replaces.

C2: 1M x 128 f32 rows, L2, a Vamana graph built on the device (R = 64, L_build = 100), 10K queries, L = 100.  In one
process, on the index's stream:
  * dab_paged_search_begin, then pages 1 .. --pages of k = 10 (dab_paged_search_next), each call timed on the host
    around the call, which returns only after the device has finished and the page is in host memory;
  * dab_search_batch(k = 10, L = 100), the first page's one-shot twin;
  * dab_search_batch(k = 100, L = 100), one search that returns as many results as ten pages.
--store picks the traversal store (default fp, full precision): sq (SQ-8), minmax (MinMax-8 behind DoubleHadamard) or
pq (PQ-32 trained on 100K rows with dab_pq_train); the session is then dab_paged_search_begin_{sq,minmax,pq}, the
one-shot twins the store's dab_search_batch_{sq,minmax,pq} without rerank, and a comparison reads the store's code row.
Every timed call runs --reps times after one warm-up (a new session each time for the paged arm); the median is
reported.  Also reported: the device memory a session holds per query (cudaMemGetInfo before begin, after begin and
after the last page), and the bytes the traversal reads per query from the cumulative cmps / hops (a 512-byte row per
comparison, a 4 * (max_degree + 1)-byte adjacency row per hop).  The card's name and power limit are read in the same
run.
usage: python tools/bench_paged.py [--n N] [--nq NQ] [--pages P] [--reps R] [--store {fp,pq,sq,minmax}] [--json PATH]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch

import bench
import diskann_b200 as dab
from bench_minmax_search import build_index, card

K, L = 10, 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=0)
    ap.add_argument("--nq", type=int, default=0)
    ap.add_argument("--pages", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--store", choices=["fp", "pq", "sq", "minmax"], default="fp")
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    name, power = card()
    cfg = dict(bench.WORKLOADS["c2_1Mx128_f32_l2"])
    n, nq = args.n or cfg["n"], args.nq or cfg["nq"]
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    g, base, centers = build_index(cfg, n, stream)
    queries = bench.make_data(cfg, bench.SEED_QUERY, nq, centers)
    dim = cfg["dim"]
    row_bytes, adj_bytes = dim * 4, 4 * (g.max_degree + 1)
    begin, one_shot = g.paged_search, g.search_batch
    if args.store == "sq":
        mean, std = base.mean(0).astype(np.float32), float(base.std())
        shift = (mean - np.float32(2.5 * std)).astype(np.float32)
        g.upload_sq(8, shift, float(np.float32(5.0 * std)), float(np.dot(shift, shift)), 0.0)
        g.sq_encode_all()
        begin, one_shot, row_bytes = g.paged_search_sq, g.search_batch_sq, dim
    elif args.store == "minmax":
        g.upload_minmax(8, 1.0, dab.Transform.double_hadamard(dim, "same", seed=7))
        g.minmax_encode_all()
        begin, one_shot, row_bytes = g.paged_search_minmax, g.search_batch_minmax, dim + 16
    elif args.store == "pq":
        sample = np.sort(np.random.default_rng(bench.SEED_PQ).choice(n, size=min(100_000, n), replace=False))
        g.pq_train(base[sample].astype(np.float32), 32, 256, 5, bench.SEED_PQ)
        g.pq_encode_all()
        begin, one_shot, row_bytes = g.paged_search_pq, g.search_batch_pq, 32

    def timed(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        return (time.perf_counter() - t) * 1e3, out

    def session():
        free0 = torch.cuda.mem_get_info()[0]
        t_begin, s = timed(lambda: begin(queries, L))
        free1 = torch.cuda.mem_get_info()[0]
        pages = [timed(lambda: s.next_page(K)) for _ in range(args.pages)]
        free2 = torch.cuda.mem_get_info()[0]
        s.close()
        return t_begin, pages, (free0 - free1) / nq, (free0 - free2) / nq

    session()  # warm-up
    runs = [session() for _ in range(args.reps)]
    last = runs[-1][1]
    page_ms = [statistics.median(r[1][p][0] for r in runs) for p in range(args.pages)]
    cmps, hops = last[-1][1][3].astype(np.float64), last[-1][1][4].astype(np.float64)
    one = {}
    for k in (K, K * args.pages):
        one_shot(queries, k, L)  # warm-up
        t = [timed(lambda: one_shot(queries, k, L)) for _ in range(args.reps)]
        r = t[-1][1]
        one[k] = dict(ms=round(statistics.median(x[0] for x in t), 3), mean_cmps=round(float(r[3].mean()), 1),
                      mean_hops=round(float(r[4].mean()), 1),
                      mb_per_query=round(float((r[3] * row_bytes + r[4] * adj_bytes).mean()) / 1e6, 4))
    # the pages' results: disjoint per query, each of k = 10
    ids = np.concatenate([p[1][0] for p in last], 1)
    distinct = all(len(set(row.tolist())) == ids.shape[1] for row in ids)
    summary = dict(
        gpu=name, power_limit_max_sm_clock=power, workload="c2_1Mx128_f32_l2", n=n, nq=nq, L=L, k=K, reps=args.reps,
        paged=dict(begin_ms=round(statistics.median(r[0] for r in runs), 3), page_ms=[round(x, 3) for x in page_ms],
                   total_ms=round(statistics.median(r[0] + sum(p[0] for p in r[1]) for r in runs), 3),
                   session_mb_per_query_after_begin=round(statistics.median(r[2] for r in runs) / 1e6, 4),
                   session_mb_per_query_after_last_page=round(statistics.median(r[3] for r in runs) / 1e6, 4),
                   mean_cmps_after_last_page=round(float(cmps.mean()), 1), mean_hops_after_last_page=round(float(hops.mean()), 1),
                   algorithmic_mb_per_query=round(float((cmps * row_bytes + hops * adj_bytes).mean()) / 1e6, 4),
                   pages_disjoint=bool(distinct)),
        search_batch_k10=one[K], search_batch_k100=one[K * args.pages])
    if args.store != "fp":
        summary["store"] = {"pq": "pq32_dab_pq_train", "sq": "sq8", "minmax": "minmax8_doublehadamard"}[args.store]
    print(json.dumps(summary), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    g.close()


if __name__ == "__main__":
    main()
