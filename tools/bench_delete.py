"""Deletes on the C2 workload of bench.py: the cost of searching with tombstones, consolidation, and the recall before
and after it.

C2: 1M x 128 f32 rows, L2, a Vamana graph built on the device (R = 64, L_build = 100), 10K queries, L = 100, k = 10.
The graph is built once and re-uploaded before each setting.  For each fraction of points deleted at random (--fracs):
  * ms of dab_delete and dab_consolidate (host clock around the call, which returns after the device has finished),
    and the lists dab_consolidate rewrote;
  * ms per batch and QPS of dab_search_batch on the same index without tombstones, with tombstones, and after
    consolidation (median of --reps after one warm-up);
  * recall@10 against exact ground truth over the live points — an exhaustive scan on the device with torch (f32, no
    TF32) in which deleted rows never qualify — with tombstones and after consolidation;
  * mean cmps and hops per query without tombstones and after consolidation.
The card's name and power limit are read in the same run.
usage: python tools/bench_delete.py [--n N] [--nq NQ] [--fracs 0.01,0.05,0.2] [--reps R] [--json PATH]"""
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
from bench_minmax_search import build_index, card

K, L = 10, 100


def ground_truth(base, queries, deleted):
    """exact top-K over the live rows (squared L2), on the device"""
    torch.backends.cuda.matmul.allow_tf32 = False
    x = torch.from_numpy(base).cuda()
    xn = (x * x).sum(1)
    dead = torch.from_numpy(deleted).cuda()
    out = []
    for q0 in range(0, queries.shape[0], 1024):
        q = torch.from_numpy(queries[q0:q0 + 1024]).cuda()
        d = (q * q).sum(1, keepdim=True) - 2.0 * q @ x.T + xn[None, :]
        d[:, dead] = float("inf")
        out.append(torch.topk(d, K, dim=1, largest=False).indices.cpu().numpy())
    return np.concatenate(out)


def recall(gt, res):
    return float(np.mean([len(np.intersect1d(gt[i], res[i][res[i] != 0xFFFFFFFF])) for i in range(gt.shape[0])]) / K)


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=0)
    ap.add_argument("--nq", type=int, default=0)
    ap.add_argument("--fracs", default="0.01,0.05,0.2")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    name, power = card()
    cfg = dict(bench.WORKLOADS["c2_1Mx128_f32_l2"])
    n, nq = args.n or cfg["n"], args.nq or cfg["nq"]
    stream = torch.cuda.Stream()
    t = time.perf_counter()
    g, base, centers = build_index(cfg, n, stream)
    build_s = time.perf_counter() - t
    queries = bench.make_data(cfg, bench.SEED_QUERY, nq, centers)
    adj0 = g.download_graph()
    rng = np.random.default_rng(7)
    search = lambda: g.search_batch(queries, K, L)  # noqa: E731
    ms_plain, plain = timed(search, args.reps)
    results = []
    for frac in (float(f) for f in args.fracs.split(",")):
        g.upload_graph(adj0)
        ids = np.sort(rng.choice(n, int(frac * n), replace=False)).astype(np.uint32)
        deleted = np.zeros(n, bool)
        deleted[ids] = True
        gt = ground_truth(base, queries, deleted)
        t = time.perf_counter()
        g.delete(ids)
        ms_delete = (time.perf_counter() - t) * 1e3
        ms_tomb, tomb = timed(search, args.reps)
        assert np.array_equal(tomb[3], plain[3]) and np.array_equal(tomb[4], plain[4])  # the traversal does not change
        t = time.perf_counter()
        rewritten = g.consolidate(cfg["R"], bench.ALPHA)
        ms_cons = (time.perf_counter() - t) * 1e3
        ms_after, after = timed(search, args.reps)
        r = {"frac": frac, "deleted": int(len(ids)), "ms_delete": ms_delete, "ms_consolidate": ms_cons, "lists_rewritten": rewritten,
             "ms_per_batch_no_tombstones": ms_plain, "ms_per_batch_tombstones": ms_tomb, "ms_per_batch_consolidated": ms_after,
             "qps_no_tombstones": nq / ms_plain * 1e3, "qps_tombstones": nq / ms_tomb * 1e3, "qps_consolidated": nq / ms_after * 1e3,
             "recall10_tombstones": recall(gt, tomb[0]), "recall10_consolidated": recall(gt, after[0]),
             "cmps_no_tombstones": float(plain[3].mean()), "hops_no_tombstones": float(plain[4].mean()),
             "cmps_consolidated": float(after[3].mean()), "hops_consolidated": float(after[4].mean())}
        results.append(r)
        print(json.dumps(r), flush=True)
        g.release(ids)
    out = {"card": name, "power_limit_and_max_sm_clock": power, "n": n, "nq": nq, "k": K, "L": L, "R": cfg["R"],
           "build_s": build_s, "settings": results}
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    g.close()


if __name__ == "__main__":
    main()
