"""Graph checks and the final prune on the C2 workload of bench.py: what dab_count_reachable and dab_degree_stats cost
against what a user does without them (dab_download_graph + a walk on the host), and what dab_prune_range does to the
graph and to search.

C2: 1M x 128 f32 rows, L2, a Vamana graph built on the device (R = 64, max_degree 83, L_build = 100), 10K queries.
  1. dab_count_reachable from the start point and dab_degree_stats over every id, timed with CUDA events around the call
     (the call returns with its result) after a warm-up, median of --reps; each against dab_download_graph plus the same
     computation on the host (a breadth-first walk with scipy's csgraph over a CSR built from the download; the degree
     statistics with numpy), timed with the host clock, with the host's results compared to the device's.
  2. The BFS kernels' time (torch.profiler, summed over bfs_seed_kernel and bfs_expand_kernel of one call) and its
     algorithmic bytes, reachable rows x adj_stride x 4 + the visited bitmap, as a share of 3.35 TB/s.
  3. Degree stats before and after dab_prune_range over every id at pruned_degree R, alpha 1.2, and search at L = 100
     on both graphs: recall@10 against exact ground truth, mean cmps and hops, and QPS with two batches in flight.
--c5 N: step 1 also on a random graph of N points at C5's adjacency shape (max_degree 83, lengths uniform in [0, 83]),
generated on the device, device calls only (the host walk is not run there).  The card's name and power limit are read
in the same run.
usage: python tools/bench_graph_stats.py [--n N] [--nq NQ] [--reps R] [--c5 N] [--json PATH]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import bench
import diskann_b200 as dab
from bench_delete import ground_truth, recall
from bench_minmax_search import build_index, card

K, L = 10, 100
HBM_BYTES_PER_S = 3.35e12
SLOT_QUERIES = 2500


def event_ms(stream, fn, reps):
    """median ms of fn() between CUDA events on `stream`, after one warm-up call"""
    out = fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        out = fn()
        b.record(stream)
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), out


def bfs_kernel_ms(fn):
    """device time of the BFS kernels of one fn() call"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = 0.0
    for e in prof.key_averages():
        if "bfs_" in e.key:
            us += getattr(e, "device_time_total", None) or e.cuda_time_total
    return us / 1e3


def host_walk(g, start):
    """dab_download_graph, then the degree statistics and a breadth-first walk on the host: (ms of download + walk, ms of
    the download, reachable, ms of download + statistics, the statistics)"""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import breadth_first_order
    t = time.perf_counter()
    adj = g.download_graph()
    t_down = time.perf_counter() - t
    n = adj.shape[0]
    deg = np.minimum(adj[:, 0], adj.shape[1] - 1)
    t_stats = time.perf_counter()
    stats = (int(deg.max()), np.float32(int(deg.sum(dtype=np.uint64))) / np.float32(n), int(deg.min()), int((deg < 2).sum()))
    t_stats = time.perf_counter() - t_stats
    mask = np.arange(adj.shape[1] - 1)[None, :] < deg[:, None]
    indptr = np.concatenate([[0], np.cumsum(deg, dtype=np.int64)])
    graph = csr_matrix((np.ones(int(indptr[-1]), np.int8), adj[:, 1:][mask].astype(np.int32), indptr), shape=(n, n))
    reached = len(breadth_first_order(graph, start, directed=True, return_predecessors=False))
    return (time.perf_counter() - t - t_stats) * 1e3, t_down * 1e3, reached, (t_down + t_stats) * 1e3, stats


def checks(g, stream, n_total, max_degree, reps, walk):
    adj_stride = (max_degree + 1 + 7) // 8 * 8
    ms_count, count = event_ms(stream, g.count_reachable, reps)
    ms_stats, stats = event_ms(stream, g.degree_stats, reps)
    k_ms = bfs_kernel_ms(g.count_reachable)
    bytes_ = count * adj_stride * 4 + (n_total + 31) // 32 * 4
    r = {"n_total": n_total, "reachable": count, "ms_count_reachable": ms_count, "ms_degree_stats": ms_stats,
         "degree_stats": {"max": stats[0], "avg": float(stats[1]), "min": stats[2], "less_than_two": stats[3]},
         "bfs_kernel_ms": k_ms, "bfs_algorithmic_bytes": bytes_,
         "bfs_share_of_3.35TBps": bytes_ / (k_ms * 1e-3) / HBM_BYTES_PER_S if k_ms > 0 else None}
    if walk:
        ms_host, ms_down, reached, ms_host_stats, host_stats = host_walk(g, n_total - 1)
        r.update({"ms_download_plus_host_walk": ms_host, "ms_download_graph": ms_down, "host_reachable": reached,
                  "host_equals_device": reached == count, "speedup_count_vs_host": ms_host / ms_count,
                  "ms_download_plus_host_degree_stats": ms_host_stats,
                  "host_degree_stats_equal_device": bool(host_stats[0] == stats[0] and host_stats[2] == stats[2] and host_stats[3] == stats[3]
                                                         and host_stats[1].view(np.uint32) == np.float32(stats[1]).view(np.uint32)),
                  "speedup_degree_stats_vs_host": ms_host_stats / ms_stats})
    print(json.dumps(r), flush=True)
    return r


def in_flight_qps(g, queries, reps):
    """QPS with two batches of SLOT_QUERIES in flight on slots 0 and 1; the last pass's results"""
    nq = queries.shape[0]
    chunks = [queries[i:i + SLOT_QUERIES] for i in range(0, nq, SLOT_QUERIES)]

    def run():
        outs, pending = [None] * len(chunks), {}
        for i, q in enumerate(chunks):
            s = i % 2
            if s in pending:
                g.wait(s)
                j, o = pending.pop(s)
                outs[j] = o
            pending[s] = (i, g.search_batch_async(s, q, K, L))
        for s, (j, o) in pending.items():
            g.wait(s)
            outs[j] = o
        return [np.concatenate([o[f] for o in outs]) for f in range(5)]

    run()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        out = run()
        ts.append(time.perf_counter() - t)
    return nq / float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=0)
    ap.add_argument("--nq", type=int, default=0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--c5", type=int, default=0)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    name, power = card()
    cfg = dict(bench.WORKLOADS["c2_1Mx128_f32_l2"])
    n, nq, R = args.n or cfg["n"], args.nq or cfg["nq"], cfg["R"]
    max_degree = bench.max_degree(R)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    g, base, centers = build_index(cfg, n, stream)
    queries = bench.make_data(cfg, bench.SEED_QUERY, nq, centers)
    out = {"card": name, "power_limit_and_max_sm_clock": power, "n": n, "nq": nq, "R": R, "max_degree": max_degree, "k": K, "L": L}
    out["c2_checks"] = checks(g, stream, n + 1, max_degree, args.reps, True)
    gt = ground_truth(base, queries, np.zeros(n, bool))

    def quality():
        qps, got = in_flight_qps(g, queries, args.reps)
        return {"recall10": recall(gt, got[0]), "qps_in_flight": qps, "cmps": float(got[3].mean()), "hops": float(got[4].mean()),
                "cmps_per_hop": float(got[3].sum() / max(1, got[4].sum()))}

    before = {"degree_stats": list(map(float, g.degree_stats())), "search": quality()}
    t = time.perf_counter()
    rewritten = g.prune_range(None, R, bench.ALPHA)
    ms_prune = (time.perf_counter() - t) * 1e3
    after = {"degree_stats": list(map(float, g.degree_stats())), "search": quality()}
    out["prune_range"] = {"pruned_degree": R, "alpha": bench.ALPHA, "ms": ms_prune, "lists_rewritten": rewritten,
                          "before": before, "after": after}
    print(json.dumps({"prune_range": out["prune_range"]}), flush=True)
    g.close()
    if args.c5:
        n5 = args.c5
        with dab.GpuIndex(dab.DType.f32, dab.Metric.L2, 4, n5, 1, max_degree) as g5:
            g5.set_stream(stream.cuda_stream)
            stride = max_degree + 1
            gen = torch.Generator(device="cuda").manual_seed(5)
            step = 1 << 22
            for first in range(0, n5 + 1, step):
                m = min(step, n5 + 1 - first)
                block = torch.randint(0, n5 + 1, (m, stride), device="cuda", dtype=torch.int64, generator=gen)
                block[:, 0] = torch.randint(0, max_degree + 1, (m,), device="cuda", generator=gen)
                block = block.to(torch.int32).contiguous()
                torch.cuda.current_stream().synchronize()
                g5.upload_graph_device(block.data_ptr(), stride, m, first)
            out["c5_shape_checks"] = checks(g5, stream, n5 + 1, max_degree, args.reps, False)
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
