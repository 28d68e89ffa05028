"""Filtered search on the C2 workload of bench.py, against the k-NN search at the same L.

C2: 1M x 128 f32 rows, L2, a Vamana graph built on the device (R = 64, L_build = 100), 10K queries, L = 100, k = 10.
Every id (the start point too) gets one random label bit, set with probability 1, 0.1 or 0.01 (the selectivity), and
every query asks for that bit (ANY).  For each selectivity, without adaptive L and with AdaptiveL(1000, 8),
dab_search_batch_filtered_device runs --reps times after two warm-up calls, timed with CUDA events around each call
(which returns with the outputs complete); the median is reported with QPS, mean cmps, hops and result count.
dab_search_batch_device on the same index and queries is timed the same way.  Filtered recall@10 is measured against
exact filtered ground truth: on the GPU, every query's L2 distance to all rows (torch, f32) with the rows the filter
rejects masked to +inf, the 10 nearest (fewer where fewer rows match); per query the share of it the search returns.
--store runs the search over a compressed store as well (the stores of bench_range.py: pq, PQ-32 trained on the device;
sq, SQ-8; minmax, MinMax-8 behind DoubleHadamard) with dab_search_batch_filtered_{pq,sq,minmax}_device, and --rerank its
full-precision rerank.  Each selectivity and adaptive setting then has a row for the store next to the full-precision
row, timed the same way, with its filtered recall@10 against the same exact ground truth and its time over that of
dab_search_batch_{pq,sq,minmax}_device (same rerank) at the same L.
The card's name and power limit are read in the same run.
usage: python tools/bench_filtered.py [--n N] [--nq NQ] [--reps R] [--store {fp,pq,sq,minmax}] [--rerank] [--json PATH]"""
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
from bench_range import build_store

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
    ap.add_argument("--store", choices=["fp", "pq", "sq", "minmax"], default="fp")
    ap.add_argument("--rerank", action="store_true")
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
    build_store(g, cfg, base, args.store)
    stores = ["fp"] if args.store == "fp" else ["fp", args.store]
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

    def knn_call(store):
        if store == "fp":
            return lambda: g.search_batch_device(d_q.data_ptr(), nq, K, L, 1, *ptrs)
        return lambda: getattr(g, f"search_batch_{store}_device")(d_q.data_ptr(), nq, K, L, 1, *ptrs, rerank=args.rerank)

    def filtered_call(store, adaptive):
        if store == "fp":
            return lambda: g.search_batch_filtered_device(d_q.data_ptr(), nq, K, L, 1, d_m.data_ptr(), *ptrs, adaptive_l=adaptive)
        return lambda: getattr(g, f"search_batch_filtered_{store}_device")(d_q.data_ptr(), nq, K, L, 1, d_m.data_ptr(), *ptrs,
                                                                           adaptive_l=adaptive, rerank=args.rerank)

    knns = {}
    truth, tcount = filtered_truth(base_t, queries, np.ones(n, bool))
    for store in stores:
        knn, kres = timed(knn_call(store))
        knn.update(store=store, rerank=args.rerank and store != "fp", recall_at_10=recall(kres, truth, tcount))
        print(json.dumps(knn), flush=True)
        knns[store] = knn
    rows = []
    rng = np.random.default_rng(0xF17E)
    for sel in SELECTIVITY:
        labels = (rng.random(n + 1) < sel).astype(np.uint64)
        g.upload_labels(labels)
        truth, tcount = filtered_truth(base_t, queries, labels[:n].astype(bool))
        for adaptive in ADAPTIVE:
            for store in stores:
                r, res = timed(filtered_call(store, adaptive))
                r.update(store=store, rerank=args.rerank and store != "fp", selectivity=sel, adaptive_l=list(adaptive) if adaptive else None,
                         filtered_recall_at_10=recall(res, truth, tcount),
                         ms_vs_knn=round(r["ms_per_batch"] / knns[store]["ms_per_batch"], 3))
                print(json.dumps(r), flush=True)
                rows.append(r)
    summary = dict(gpu=name, power_limit_max_sm_clock=power, workload="c2_1Mx128_f32_l2", n=n, nq=nq, L=L, k=K, reps=args.reps,
                   store={"fp": "full_precision", "pq": "pq32_dab_pq_train", "sq": "sq8", "minmax": "minmax8_doublehadamard"}[args.store],
                   rerank=args.rerank, search_batch=knns["fp"], search_batch_store=knns.get(args.store), filtered=rows)
    print(json.dumps(summary), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    g.close()


if __name__ == "__main__":
    main()
