"""Filtered search on the C2 workload of bench.py, against the k-NN search at the same L.

C2: 1M x 128 f32 rows, L2, a Vamana graph built on the device (R = 64, L_build = 100), 10K queries, L = 100, k = 10.
Every id (the start point too) gets one random label bit, set with probability 1, 0.1 or 0.01 (the selectivity), and
every query asks for that bit (ANY).  For each selectivity, without adaptive L and with AdaptiveL(1000, 8),
dab_search_batch_filtered_device runs --reps times after two warm-up calls, timed with CUDA events around each call
(which returns with the outputs complete); the median is reported with QPS, mean cmps, hops and result count.
dab_search_batch_device on the same index and queries is timed the same way.  Filtered recall@10 is measured against
exact filtered ground truth: on the GPU, every query's L2 distance to all rows (torch, f32) with the rows the filter
rejects masked to +inf, the 10 nearest (fewer where fewer rows match); per query the share of it the search returns.
The card's name and power limit are read in the same run.
usage: python tools/bench_filtered.py [--n N] [--nq NQ] [--reps R] [--json PATH]"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch

import bench
import diskann_b200 as dab
from bench_minmax_search import build_index, card

K, L = 10, 100
SELECTIVITY = (1.0, 0.1, 0.01)
ADAPTIVE = (None, (1000, 8.0))


def filtered_truth(base_t, queries, accept):
    """per query the ids of the K nearest accepted rows by L2 (torch, f32), nearest first, and how many there are"""
    bn = (base_t * base_t).sum(1)
    rejected = ~torch.from_numpy(accept).cuda()
    ids, cnt = [], []
    for q0 in range(0, queries.shape[0], 256):
        q = torch.from_numpy(queries[q0:q0 + 256]).cuda()
        d = bn[None, :] - 2.0 * (q @ base_t.T) + (q * q).sum(1, keepdim=True)
        d[:, rejected] = float("inf")
        v, i = torch.topk(d, K, dim=1, largest=False, sorted=True)
        ids.append(i.cpu().numpy())
        cnt.append(torch.isfinite(v).sum(1).cpu().numpy())
    return np.concatenate(ids), np.concatenate(cnt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=0)
    ap.add_argument("--nq", type=int, default=0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    name, power = card()
    cfg = dict(bench.WORKLOADS["c2_1Mx128_f32_l2"])
    n, nq = args.n or cfg["n"], args.nq or cfg["nq"]
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    g, base, centers = build_index(cfg, n, stream)
    queries = bench.make_data(cfg, bench.SEED_QUERY, nq, centers)
    base_t = torch.from_numpy(base).cuda()
    d_q = torch.from_numpy(queries).cuda()
    d_m = torch.ones(nq, dtype=torch.int64, device="cuda")  # every query asks for bit 0
    outs = (torch.empty((nq, K), dtype=torch.int32, device="cuda"), torch.empty((nq, K), dtype=torch.float32, device="cuda"),
            *(torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3)))
    ptrs = [o.data_ptr() for o in outs]

    def timed(call):
        call()
        call()
        ms = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            call()
            b.record(stream)
            b.synchronize()
            ms.append(a.elapsed_time(b))
        res = [o.cpu().numpy() for o in outs]
        t = statistics.median(ms)
        return dict(ms_per_batch=round(t, 3), qps=round(nq / t * 1e3, 1), mean_cmps=round(float(res[3].mean()), 1),
                    mean_hops=round(float(res[4].mean()), 1), mean_count=round(float(res[2].mean()), 2)), res

    def recall(res, truth, tcount):
        ids, counts = res[0].view(np.uint32), res[2]
        got = [len(np.intersect1d(truth[q, :tcount[q]], ids[q, :counts[q]])) / tcount[q] for q in range(nq) if tcount[q]]
        return round(float(np.mean(got)), 4) if got else None

    knn, kres = timed(lambda: g.search_batch_device(d_q.data_ptr(), nq, K, L, 1, *ptrs))
    truth, tcount = filtered_truth(base_t, queries, np.ones(n, bool))
    knn["recall_at_10"] = recall(kres, truth, tcount)
    print(json.dumps(knn), flush=True)
    rows = []
    rng = np.random.default_rng(0xF17E)
    for sel in SELECTIVITY:
        labels = (rng.random(n + 1) < sel).astype(np.uint64)
        g.upload_labels(labels)
        truth, tcount = filtered_truth(base_t, queries, labels[:n].astype(bool))
        for adaptive in ADAPTIVE:
            r, res = timed(lambda: g.search_batch_filtered_device(d_q.data_ptr(), nq, K, L, 1, d_m.data_ptr(), *ptrs, adaptive_l=adaptive))
            r.update(selectivity=sel, adaptive_l=list(adaptive) if adaptive else None, filtered_recall_at_10=recall(res, truth, tcount),
                     ms_vs_knn=round(r["ms_per_batch"] / knn["ms_per_batch"], 3))
            print(json.dumps(r), flush=True)
            rows.append(r)
    summary = dict(gpu=name, power_limit_max_sm_clock=power, workload="c2_1Mx128_f32_l2", n=n, nq=nq, L=L, k=K, reps=args.reps,
                   search_batch=knn, filtered=rows)
    print(json.dumps(summary), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    g.close()


if __name__ == "__main__":
    main()
