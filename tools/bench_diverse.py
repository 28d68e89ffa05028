"""Diverse search on the C2 workload of bench.py, against the k-NN search at the same L.

C2: 1M x 128 f32 rows, L2, a Vamana graph built on the device (R = 64, L_build = 100), 10K queries, L = 100, k = 10.
Every id (the start point too) gets a uniform random attribute out of 5, 1000 or n / 10 values; for each cardinality and
diverse_k of 1 and 3, dab_search_batch_diverse_device runs --reps times after two warm-up calls, timed with CUDA events
around each call (which returns with the outputs complete); the median is reported with QPS, mean cmps and hops.
dab_search_batch_device at the same L is timed the same way.  Diverse recall@10 is measured against exact ground truth:
all points sorted by exact distance (the 4096 nearest, computed on the GPU with torch, and the whole sorted list for a
query whose 4096 nearest do not hold enough values), at most diverse_k per attribute value, the first 10; per query the
share of its ground truth (10, or fewer when the cardinality allows fewer) the search returns.  The diversity bound is
checked on every result row: the largest number of results that share an attribute value, and the queries where it
exceeds diverse_k (the reference's tie drift may allow that; it is reported as measured).  Those queries are searched
again by the CPU oracle (orc_search_batch_diverse over the downloaded graph): whether it returns the same ids, distance
bits, counts, cmps and hops, and how many of its queue removals failed on an exact distance tie; over the PQ and MinMax
stores the first 16 of them, by orc_search_batch_diverse_table fed the store's distances to every id (the SQ store is not
checked: its restatement holds every row's codes unpacked, too large at C2).  The k-NN batch's recall@10 against the
nearest 10 is reported with it.  The card's name and power limit are read in the same run.
--store picks the traversal store (default fp, full precision): sq (SQ-8), minmax (MinMax-8 behind DoubleHadamard) or
pq (PQ-32 trained on 100K rows with dab_pq_train), as tools/bench_paged.py sets them up; the calls are then
dab_search_batch_diverse_{sq,minmax,pq}_device and dab_search_batch_{sq,minmax,pq}_device, with --rerank the
full-precision rerank of both.  Each diverse row also reports its re-run passes: the kernel launches of one call beyond
those of a call that re-runs nothing (the fewest launches of four one-query calls), and an upper bound on the queries
whose visited table can have overflowed (final visited set = cmps, plus max_degree, past 7/8 of the first pass's table).
usage: python tools/bench_diverse.py [--n N] [--nq NQ] [--reps R] [--store {fp,pq,sq,minmax}] [--rerank] [--json PATH]"""
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

sys.path.insert(0, os.path.join(ROOT, "tests"))
import diverse_oracle  # noqa: E402  the CPU checker of the queries over diverse_k
import diverse_table_oracle  # noqa: E402  ... and over a quantized store's distances
import oracle_lib  # noqa: E402

K, L, TOP = 10, 100, 4096
OVER_SAMPLE = 16  # quantized stores: the queries over diverse_k the oracle checks


def nearest(base_t, queries, top):
    """ids of the `top` nearest rows of every query by L2 (torch, f32), nearest first"""
    out = []
    bn = (base_t * base_t).sum(1)
    for q0 in range(0, queries.shape[0], 256):
        q = torch.from_numpy(queries[q0:q0 + 256]).cuda()
        d = bn[None, :] - 2.0 * (q @ base_t.T) + (q * q).sum(1, keepdim=True)
        out.append(torch.topk(d, top, dim=1, largest=False, sorted=True).indices.cpu().numpy())
    return np.concatenate(out)


def diverse_truth(order, attrs, dk, want):
    """per row of `order` (ids nearest first): the first `want` ids with at most dk per attribute value; rows that run
    out of ids are returned as None"""
    a = attrs[order].astype(np.int64)
    srt = np.argsort(a, axis=1, kind="stable")
    sa = np.take_along_axis(a, srt, 1)
    start = np.maximum.accumulate(np.where(np.diff(sa, axis=1, prepend=-1) != 0, np.arange(a.shape[1])[None, :], 0), axis=1)
    occ = np.empty_like(srt)
    np.put_along_axis(occ, srt, np.arange(a.shape[1])[None, :] - start, 1)
    keep = occ < dk
    out = []
    for r in range(order.shape[0]):
        ids = order[r][keep[r]][:want]
        out.append(ids if ids.shape[0] == want else None)
    return out


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
    order = nearest(base_t, queries, min(TOP, n))
    d_q = torch.from_numpy(queries).cuda()
    outs = (torch.empty((nq, K), dtype=torch.int32, device="cuda"), torch.empty((nq, K), dtype=torch.float32, device="cuda"),
            *(torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3)))
    ptrs = [o.data_ptr() for o in outs]
    dim = cfg["dim"]
    if args.store == "sq":
        mean, std = base.mean(0).astype(np.float32), float(base.std())
        shift = (mean - np.float32(2.5 * std)).astype(np.float32)
        g.upload_sq(8, shift, float(np.float32(5.0 * std)), float(np.dot(shift, shift)), 0.0)
        g.sq_encode_all()
    elif args.store == "minmax":
        g.upload_minmax(8, 1.0, dab.Transform.double_hadamard(dim, "same", seed=7))
        g.minmax_encode_all()
    elif args.store == "pq":
        sample = np.sort(np.random.default_rng(bench.SEED_PQ).choice(n, size=min(100_000, n), replace=False))
        g.pq_train(base[sample].astype(np.float32), 32, 256, 5, bench.SEED_PQ)
        g.pq_encode_all()
    rr = dict(rerank=args.rerank)

    stores = {}

    def store_distances(q):
        """the store's traversal distance of query q to every id (the quantizer restated on the CPU, as the tests do)"""
        from test_paged_search_quantized import PQStore
        if args.store == "minmax":
            from test_minmax_search import compress
            if "rows" not in stores:
                stores["rows"] = g.download_minmax()
            rows = stores["rows"]
            qr = compress(q[None], dab.Transform.double_hadamard(dim, "same", seed=7), 8)[0]
            return oracle_lib.minmax_distances(oracle_lib.L2, 8, 8, np.broadcast_to(qr, rows.shape), rows)
        if "st" not in stores:
            stores["st"] = PQStore(*g.download_pq(), oracle_lib.L2)
        return stores["st"].distances(q)

    def knn_call():
        if args.store == "fp":
            g.search_batch_device(d_q.data_ptr(), nq, K, L, 1, *ptrs)
        else:
            getattr(g, f"search_batch_{args.store}_device")(d_q.data_ptr(), nq, K, L, 1, *ptrs, **rr)

    def diverse_call(dk, q_ptr=None, m=None):
        q_ptr, m = q_ptr or d_q.data_ptr(), m or nq
        if args.store == "fp":
            g.search_batch_diverse_device(q_ptr, m, K, L, dk, 1, *ptrs)
        else:
            getattr(g, f"search_batch_diverse_{args.store}_device")(q_ptr, m, K, L, dk, 1, *ptrs, **rr)

    def launches(call):
        before = dab.launch_count()
        call()
        stream.synchronize()
        return dab.launch_count() - before

    # the first pass's visited table (table_slots without a hint: 1.1 * max_degree * 1.3 * L) and its 7/8 limit
    hlimit = (max(256, int(1.1 * g.max_degree * 1.3 * L) + 1) + 7) // 8 * 7

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
                    mean_hops=round(float(res[4].mean()), 1)), res

    knn, kres = timed(knn_call)
    kids = kres[0].view(np.uint32)
    knn["recall_at_10"] = round(float(np.mean([len(np.intersect1d(order[qi, :K], kids[qi, :kres[2][qi]])) / K for qi in range(nq)])), 4)
    rows = []
    oracle = None
    rng = np.random.default_rng(0xD1CE)
    for card_n in (5, 1000, n // 10):
        attrs = rng.integers(0, card_n, n + 1).astype(np.uint32)
        g.upload_attributes(attrs)
        for dk in (1, 3):
            r, res = timed(lambda: diverse_call(dk))
            base_launches = min(launches(lambda: diverse_call(dk, d_q[i:i + 1].data_ptr(), 1)) for i in range(4))
            r.update(rerun_passes=launches(lambda: diverse_call(dk)) - base_launches,
                     queries_near_visited_limit=int((res[3].astype(np.int64) + g.max_degree > hlimit).sum()))
            ids, counts = res[0].view(np.uint32), res[2]
            want = min(K, card_n * dk)
            truth = diverse_truth(order, attrs, dk, want)
            recall, full_sorts = [], 0
            for qi in range(nq):
                t = truth[qi]
                if t is None:  # the nearest TOP rows do not hold enough values: the whole list
                    full_sorts += 1
                    d = ((base - queries[qi]) ** 2).sum(1)
                    t = diverse_truth(np.argsort(d, kind="stable")[None, :], attrs, dk, want)[0]
                recall.append(len(np.intersect1d(t, ids[qi, :counts[qi]])) / want)
            worst = [int(np.bincount(attrs[ids[qi, :counts[qi]]]).max()) if counts[qi] else 0 for qi in range(nq)]
            r.update(cardinality=card_n, diverse_k=dk, diverse_recall_at_10=round(float(np.mean(recall)), 4),
                     truth_size=want, truth_full_sorts=full_sorts, mean_count=round(float(counts.mean()), 2),
                     max_results_per_value=max(worst), queries_over_diverse_k=int(sum(w > dk for w in worst)))
            over = np.array([qi for qi in range(nq) if worst[qi] > dk], np.int64)
            if over.size and args.store != "sq":
                if oracle is None:
                    vecs = np.concatenate([base, bench.find_medoid(base)[None, :]])
                    oracle = oracle_lib.Index(vecs, g.download_graph(), n, 1, oracle_lib.L2)
                if args.store == "fp":
                    want_o = diverse_oracle.search_batch(oracle, queries[over], K, L, dk, attrs)
                else:
                    over = over[:OVER_SAMPLE]  # the store's distances to every id, one query at a time
                    tables = np.stack([store_distances(q) for q in queries[over]])
                    want_o = diverse_table_oracle.search_batch_table(oracle, tables, queries[over], K, L, dk, attrs, rerank=args.rerank)
                    r.update(over_diverse_k_checked=int(over.size))
                same = all(np.array_equal(np.asarray(a)[over].view(np.uint32), np.asarray(b).view(np.uint32))
                           for a, b in zip(res, want_o[:5]))
                r.update(over_diverse_k_equal_to_oracle=bool(same), over_diverse_k_failed_removals=int(want_o[5].sum()))
            print(json.dumps(r), flush=True)
            rows.append(r)
    summary = dict(gpu=name, power_limit_max_sm_clock=power, workload="c2_1Mx128_f32_l2", n=n, nq=nq, L=L, k=K, reps=args.reps,
                   store={"fp": "full_precision", "pq": "pq32_dab_pq_train", "sq": "sq8", "minmax": "minmax8_doublehadamard"}[args.store],
                   rerank=args.rerank, search_batch=knn, diverse=rows)
    print(json.dumps(summary), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    g.close()


if __name__ == "__main__":
    main()
