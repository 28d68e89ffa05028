"""Inserts on the C2 workload of bench.py: the streaming cycle delete -> consolidate -> release -> insert, what the
inserts cost and what the graph is worth afterwards.

C2: 1M x 128 f32 rows, L2, a Vamana graph built on the device (R = 64, L_build = 100), 10K queries, L = 100, k = 10.
The graph is built once (and dab_build timed once more on it, for its points per second).  For each fraction of points
(--fracs): that many random points are deleted, the graph is consolidated and the ids released; the released graph is
then re-uploaded before each batch size of --batch, and as many fresh rows from the same distribution are inserted into
the released ids with dab_insert (pruned degree R, L_build, alpha 1.2).  Reported:
  * ms of dab_delete, dab_consolidate, dab_release and dab_insert (host clock around the call, which returns after the
    device has finished) and inserts per second;
  * recall@10 at L = 100 against exact ground truth over every row (an exhaustive scan on the device with torch, f32, no
    TF32), QPS, mean cmps and hops — before the deletes and after the re-inserts.
--parity: after one 1024-point insert, the downloaded graph is compared word for word with the oracle's
orc_insert_batched on the host.  The card's name and power limit are read in the same run.
usage: python tools/bench_insert.py [--n N] [--nq NQ] [--fracs 0.01,0.05] [--batch 1024,0] [--reps R] [--parity] [--json PATH]"""
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
from bench_delete import ground_truth, recall, timed
from bench_minmax_search import build_index, card

K, L = 10, 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=0)
    ap.add_argument("--nq", type=int, default=0)
    ap.add_argument("--fracs", default="0.01,0.05")
    ap.add_argument("--batch", default="1024,0")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parity", action="store_true")
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    name, power = card()
    cfg = dict(bench.WORKLOADS["c2_1Mx128_f32_l2"])
    n, nq, R, lb = args.n or cfg["n"], args.nq or cfg["nq"], cfg["R"], cfg["l_build"]
    stream = torch.cuda.Stream()
    g, base, centers = build_index(cfg, n, stream)
    t = time.perf_counter()
    g.build(R, lb, bench.ALPHA)  # the same graph again, timed on its own
    build_s = time.perf_counter() - t
    queries = bench.make_data(cfg, bench.SEED_QUERY, nq, centers)
    adj0 = g.download_graph()
    start = bench.find_medoid(base)[None, :]  # the start row build_index uploaded
    rng = np.random.default_rng(11)
    search = lambda: g.search_batch(queries, K, L)  # noqa: E731
    gt0 = ground_truth(base, queries, np.zeros(n, bool))
    ms0, before = timed(search, args.reps)
    stats_before = {"recall10": recall(gt0, before[0]), "qps": nq / ms0 * 1e3, "ms_per_batch": ms0,
                    "cmps": float(before[3].mean()), "hops": float(before[4].mean())}
    print(json.dumps({"before": stats_before, "build_s": build_s, "build_points_per_s": n / build_s}), flush=True)
    results, parity = [], None
    for fi, frac in enumerate(float(f) for f in args.fracs.split(",")):
        g.upload_vectors(base)
        g.upload_graph(adj0)
        ids = rng.choice(n, int(frac * n), replace=False).astype(np.uint32)
        t = time.perf_counter()
        g.delete(ids)
        ms_delete = (time.perf_counter() - t) * 1e3
        t = time.perf_counter()
        rewritten = g.consolidate(R, bench.ALPHA)
        ms_cons = (time.perf_counter() - t) * 1e3
        t = time.perf_counter()
        g.release(ids)
        ms_release = (time.perf_counter() - t) * 1e3
        released = g.download_graph()
        fresh = bench.make_data(cfg, bench.SEED_BASE + 1 + fi, len(ids), centers)
        new = base.copy()
        new[ids] = fresh
        gt = ground_truth(new, queries, np.zeros(n, bool))
        for batch in (int(b) for b in args.batch.split(",")):
            g.upload_vectors(base)
            g.upload_graph(released)
            t = time.perf_counter()
            g.insert(ids, fresh, R, lb, bench.ALPHA, batch)
            ms_insert = (time.perf_counter() - t) * 1e3
            ms_after, after = timed(search, args.reps)
            r = {"frac": frac, "points": int(len(ids)), "batch": batch, "ms_delete": ms_delete, "ms_consolidate": ms_cons,
                 "lists_rewritten": rewritten, "ms_release": ms_release, "ms_insert": ms_insert,
                 "inserts_per_s": len(ids) / ms_insert * 1e3, "recall10_after": recall(gt, after[0]), "qps_after": nq / ms_after * 1e3,
                 "ms_per_batch_after": ms_after, "cmps_after": float(after[3].mean()), "hops_after": float(after[4].mean())}
            results.append(r)
            print(json.dumps(r), flush=True)
        if args.parity and parity is None:
            import oracle_lib as O
            from insert_oracle import insert_batched
            sub = ids[:1024]
            g.upload_vectors(base)
            g.upload_graph(released)
            g.insert(sub, new[sub], R, lb, bench.ALPHA, 1024)
            got = g.download_graph()
            vecs = np.concatenate([base, start])
            vecs[sub] = new[sub]
            want = insert_batched(vecs, released, sub, n, 1, O.L2, R, bench.max_degree(R), lb, bench.ALPHA, batch_size=1024)
            parity = {"points": int(len(sub)), "rows_differing": int((got != want).any(1).sum())}
            print(json.dumps({"parity": parity}), flush=True)
    out = {"card": name, "power_limit_and_max_sm_clock": power, "n": n, "nq": nq, "k": K, "L": L, "R": R, "l_build": lb,
           "build_s": build_s, "build_points_per_s": n / build_s, "before": stats_before, "settings": results, "parity": parity}
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    g.close()


if __name__ == "__main__":
    main()
