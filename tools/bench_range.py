"""Range search on the C2 workload of bench.py, against the k-NN search at the same L.

C2: 1M x 128 f32 rows, L2, a Vamana graph built on the device (R = 64, L_build = 100), 10K queries, L = 100.  The radii
are those at which the exact mean in-range count is about 10, 100 and 1000: bisection on the radius over the exact
distances of every query to every row (f64, on the GPU with torch).  For each radius dab_range_search_device runs --reps
times after two warm-up calls, timed with CUDA events around each call (which returns with the result set complete);
the median is reported.  Phase 1 is the k-NN traversal with k = L, which dab_search_batch_device runs on its own at the
same L and beam: it is timed the same way and reported as the phase-1 time, and the rest of the range call as phase 2
(its in_range pass, second rounds, re-runs, scan and compaction).  Per radius: the mean and largest result counts, the
share of queries that took a second round, mean hops, and the reference's average_precision (benchmark-core/src/
recall.rs: the share of all exact in-range ids, over all queries, that the search returned).  The card's name and power
limit are read in the same run.
--store runs the search over a compressed store as well (the stores of bench_diverse.py: pq, PQ-32 trained on the device;
sq, SQ-8; minmax, MinMax-8 behind DoubleHadamard) with dab_range_search_{pq,sq,minmax}_device, and --rerank its
full-precision rerank.  Each radius then has a row for the store next to the full-precision row, timed the same way
(phase 1 of the store is dab_search_batch_{pq,sq,minmax}_device at L), with its average_precision against the same exact
full-precision in-range sets.
--selectivity S runs dab_range_search_filtered_device instead of the unfiltered call: bit 0 of the label table is set on
a share S of the ids (seeded draw), every query's mask is that bit (ANY), and the exact sets are the in-range ids that
carry it.  Its rows report the same numbers; phase 1 is not separated (the filtered traversal is part of the call).
With --store, each radius also has a row for dab_range_search_filtered_{pq,sq,minmax}_device (with --rerank, its
full-precision rerank) next to the fp_filtered row, with its average_precision against the same exact matching sets.
usage: python tools/bench_range.py [--n N] [--nq NQ] [--reps R] [--beam B] [--store {fp,pq,sq,minmax}] [--rerank]
                                   [--selectivity S] [--json PATH]"""
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

L, TARGETS, CHUNK = 100, (10, 100, 1000), 128


def in_range_sets(base_t, bn, queries, radius, want_ids):
    """exact in-range counts of every query (and, with want_ids, their ids) at `radius`, f64"""
    counts, ids = [], []
    for q0 in range(0, queries.shape[0], CHUNK):
        q = torch.from_numpy(queries[q0:q0 + CHUNK]).cuda().double()
        d = bn[None, :] - 2.0 * (q @ base_t.T) + (q * q).sum(1, keepdim=True)
        m = d <= radius
        counts.append(m.sum(1).cpu().numpy())
        if want_ids:
            nz = torch.nonzero(m).cpu().numpy()
            ids.extend(np.split(nz[:, 1], np.cumsum(np.bincount(nz[:, 0], minlength=m.shape[0]))[:-1]))
    return np.concatenate(counts), ids


def build_store(g, cfg, base, store):
    """the compressed store `store` of g over its rows `base` (fp: none): PQ-32 trained on the device, SQ-8, or MinMax-8
    behind DoubleHadamard"""
    n = base.shape[0]
    if store == "sq":
        mean, std = base.mean(0).astype(np.float32), float(base.std())
        shift = (mean - np.float32(2.5 * std)).astype(np.float32)
        g.upload_sq(8, shift, float(np.float32(5.0 * std)), float(np.dot(shift, shift)), 0.0)
        g.sq_encode_all()
    elif store == "minmax":
        g.upload_minmax(8, 1.0, dab.Transform.double_hadamard(cfg["dim"], "same", seed=7))
        g.minmax_encode_all()
    elif store == "pq":
        pick = np.sort(np.random.default_rng(bench.SEED_PQ).choice(n, size=min(100_000, n), replace=False))
        g.pq_train(base[pick].astype(np.float32), 32, 256, 5, bench.SEED_PQ)
        g.pq_encode_all()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=0)
    ap.add_argument("--nq", type=int, default=0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--beam", type=int, default=1)
    ap.add_argument("--store", choices=["fp", "pq", "sq", "minmax"], default="fp")
    ap.add_argument("--rerank", action="store_true")
    ap.add_argument("--selectivity", type=float, default=None)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    name, power = card()
    cfg = dict(bench.WORKLOADS["c2_1Mx128_f32_l2"])
    n, nq = args.n or cfg["n"], args.nq or cfg["nq"]
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    g, base, centers = build_index(cfg, n, stream)
    queries = bench.make_data(cfg, bench.SEED_QUERY, nq, centers)
    base_t = torch.from_numpy(base).cuda().double()
    bn = (base_t * base_t).sum(1)
    d_q = torch.from_numpy(queries).cuda()
    build_store(g, cfg, base, args.store)
    stores = ["fp"] if args.store == "fp" else ["fp", args.store]
    accepted = None
    if args.selectivity is not None:
        accepted = np.random.default_rng(bench.SEED_QUERY + 1).random(n + 1) < args.selectivity
        g.upload_labels(accepted.astype(np.uint64))
        d_masks = torch.ones(nq, dtype=torch.int64, device="cuda")
        stores = ["fp_filtered"] if args.store == "fp" else ["fp_filtered", f"{args.store}_filtered"]

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
        return statistics.median(ms)

    outs = (torch.empty((nq, L), dtype=torch.int32, device="cuda"), torch.empty((nq, L), dtype=torch.float32, device="cuda"),
            *(torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3)))
    knn_ms = timed(lambda: g.search_batch_device(d_q.data_ptr(), nq, L, L, args.beam, *(o.data_ptr() for o in outs)))
    knn_d = outs[1].cpu().numpy()
    phase1 = {"fp": knn_ms}
    if args.store != "fp":
        phase1[args.store] = timed(lambda: getattr(g, f"search_batch_{args.store}_device")(d_q.data_ptr(), nq, L, L, args.beam,
                                                                                           *(o.data_ptr() for o in outs)))

    def range_set(store, radius):
        if store == "fp_filtered":
            return g.range_search_filtered_device(d_q.data_ptr(), d_masks.data_ptr(), nq, L, radius, beam_width=args.beam)
        if store.endswith("_filtered"):
            return getattr(g, f"range_search_filtered_{args.store}_device")(d_q.data_ptr(), d_masks.data_ptr(), nq, L, radius,
                                                                            beam_width=args.beam, rerank=args.rerank)
        if store == "fp":
            return g.range_search_device(d_q.data_ptr(), nq, L, radius, beam_width=args.beam)
        return getattr(g, f"range_search_{store}_device")(d_q.data_ptr(), nq, L, radius, beam_width=args.beam, rerank=args.rerank)

    sample = queries[:: max(1, nq // 1000)]
    rows = []
    for target in TARGETS:
        lo, hi = 0.0, float(np.median(knn_d[:, -1])) * 16
        for _ in range(30):  # bisection on the mean exact count over a sample of the queries
            mid = (lo + hi) / 2
            if in_range_sets(base_t, bn, sample, mid, False)[0].mean() < target:
                lo = mid
            else:
                hi = mid
        radius = float(np.float32(hi))
        exact, truth = in_range_sets(base_t, bn, queries, radius, True)
        if accepted is not None:  # the exact matching sets
            truth = [t[accepted[t]] for t in truth]
            exact = np.array([len(t) for t in truth])

        for store in stores:
            def call():
                with range_set(store, radius):
                    pass
            ms = timed(call)
            with range_set(store, radius) as r:
                offsets, cmps, hops, second = r.offsets()
                ids, _ = r.results()
            counts = np.diff(offsets.astype(np.int64))
            found = sum(len(np.intersect1d(truth[q], ids[offsets[q]:offsets[q + 1]])) for q in range(nq))
            row = dict(store=store, rerank=args.rerank and store not in ("fp", "fp_filtered"), target_mean_count=target, radius=radius,
                       exact_mean_count=round(float(exact.mean()), 2), exact_max_count=int(exact.max()), ms_per_batch=round(ms, 3),
                       phase1_ms=round(phase1.get(store, float("nan")), 3), phase2_ms=round(ms - phase1.get(store, float("nan")), 3),
                       qps=round(nq / ms * 1e3, 1),
                       mean_count=round(float(counts.mean()), 2), max_count=int(counts.max()),
                       second_round_share=round(float(second.mean()), 4), mean_hops=round(float(hops.mean()), 1),
                       mean_cmps=round(float(cmps.mean()), 1), average_precision=round(found / max(1, int(exact.sum())), 4))
            print(json.dumps(row), flush=True)
            rows.append(row)
    summary = dict(gpu=name, power_limit_max_sm_clock=power, workload="c2_1Mx128_f32_l2", n=n, nq=nq, L=L, beam=args.beam,
                   store={"fp": "full_precision", "pq": "pq32_dab_pq_train", "sq": "sq8", "minmax": "minmax8_doublehadamard"}[args.store],
                   rerank=args.rerank, selectivity=args.selectivity, reps=args.reps, knn_batch_ms=round(knn_ms, 3), range=rows)
    print(json.dumps(summary), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    g.close()


if __name__ == "__main__":
    main()
