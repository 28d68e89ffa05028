"""In-place deletes on the C2 workload of bench.py: what dab_inplace_delete costs against dab_delete + dab_consolidate,
and what the graph is worth afterwards.

C2: 1M x 128 f32 rows, L2, a Vamana graph built on the device (R = 64, L_build = 100), 10K queries, L = 100, k = 10.
The graph is built once.  For each fraction of points (--fracs) the same random ids are deleted by every arm, each on
the built graph re-uploaded (the previous arm's marks released first):
  * dab_inplace_delete with each method (--methods) at each batch size (--batch), with the example runbooks' parameters
    (VisitedAndTopK k = 20, l = 50; num_to_replace 3; pruned degree R, alpha 1.2), then dab_drop_deleted_neighbors;
  * dab_delete + dab_consolidate.
Reported per arm: ms of each call (host clock around the call, which returns after the device has finished), deletes
per second, lists rewritten, and recall@10 at L = 100 against exact ground truth over the live points (an exhaustive
scan on the device with torch, f32, no TF32), QPS, mean cmps and hops — before the deletes, after the in-place delete (or
the consolidation) and after the drop.
--parity: one 1024-id chunk (VisitedAndTopK) on the built graph, the downloaded graph and deletion table compared word
for word with the oracle's orc_inplace_delete on the host.  The card's name and power limit are read in the same run.
usage: python tools/bench_inplace_delete.py [--n N] [--nq NQ] [--fracs 0.01,0.05] [--batch 1,0]
                                            [--methods visited_and_topk,two_hop_and_one_hop,one_hop] [--reps R] [--parity]
                                            [--json PATH]"""
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
NUM_TO_REPLACE, K_VALUE, L_VALUE = 3, 20, 50  # diskann-benchmark/example/graph-index-dynamic*.json


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=0)
    ap.add_argument("--nq", type=int, default=0)
    ap.add_argument("--fracs", default="0.01,0.05")
    ap.add_argument("--batch", default="1,0")
    ap.add_argument("--methods", default="visited_and_topk,two_hop_and_one_hop,one_hop")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parity", action="store_true")
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    name, power = card()
    cfg = dict(bench.WORKLOADS["c2_1Mx128_f32_l2"])
    n, nq, R = args.n or cfg["n"], args.nq or cfg["nq"], cfg["R"]
    stream = torch.cuda.Stream()
    g, base, centers = build_index(cfg, n, stream)
    queries = bench.make_data(cfg, bench.SEED_QUERY, nq, centers)
    adj0 = g.download_graph()
    start = bench.find_medoid(base)[None, :]  # the start row build_index uploaded
    rng = np.random.default_rng(13)
    search = lambda: g.search_batch(queries, K, L)  # noqa: E731

    def quality(gt):
        ms, got = timed(search, args.reps)
        return {"recall10": recall(gt, got[0]), "qps": nq / ms * 1e3, "ms_per_batch": ms, "cmps": float(got[3].mean()),
                "hops": float(got[4].mean())}

    before = quality(ground_truth(base, queries, np.zeros(n, bool)))
    print(json.dumps({"before": before}), flush=True)
    results, marked = [], np.zeros(0, np.uint32)

    def reset():
        nonlocal marked
        if len(marked):
            g.release(marked)
            marked = np.zeros(0, np.uint32)
        g.upload_graph(adj0)

    def ms_of(call):
        t = time.perf_counter()
        out = call()
        return (time.perf_counter() - t) * 1e3, out

    for frac in (float(f) for f in args.fracs.split(",")):
        ids = rng.choice(n, int(frac * n), replace=False).astype(np.uint32)
        dead = np.zeros(n, bool)
        dead[ids] = True
        gt = ground_truth(base, queries, dead)
        for method in args.methods.split(","):
            for batch in (int(b) for b in args.batch.split(",")):
                reset()
                ms_del, _ = ms_of(lambda: g.inplace_delete(ids, NUM_TO_REPLACE, method, R, bench.ALPHA, K_VALUE, L_VALUE, batch))
                marked = ids
                after = quality(gt)
                ms_drop, dropped = ms_of(lambda: g.drop_deleted_neighbors(R))
                r = {"frac": frac, "points": int(len(ids)), "arm": "inplace_delete", "method": method, "batch": batch,
                     "ms_call": ms_del, "deletes_per_s": len(ids) / ms_del * 1e3, "after": after,
                     "ms_drop_deleted_neighbors": ms_drop, "lists_dropped": dropped, "after_drop": quality(gt)}
                results.append(r)
                print(json.dumps(r), flush=True)
        reset()
        ms_del, _ = ms_of(lambda: g.delete(ids))
        marked = ids
        ms_cons, rewritten = ms_of(lambda: g.consolidate(R, bench.ALPHA))
        r = {"frac": frac, "points": int(len(ids)), "arm": "delete_consolidate", "ms_delete": ms_del, "ms_consolidate": ms_cons,
             "ms_call": ms_del + ms_cons, "deletes_per_s": len(ids) / (ms_del + ms_cons) * 1e3, "lists_rewritten": rewritten,
             "after": quality(gt)}
        results.append(r)
        print(json.dumps(r), flush=True)
    parity = None
    if args.parity:
        import inplace_delete_oracle as D
        import oracle_lib as O
        reset()
        sub = rng.choice(n, 1024, replace=False).astype(np.uint32)
        g.inplace_delete(sub, NUM_TO_REPLACE, "visited_and_topk", R, bench.ALPHA, K_VALUE, L_VALUE, 0)
        marked = sub
        got = g.download_graph()
        status = np.flatnonzero(g.delete_status(np.arange(n, dtype=np.uint32))).astype(np.uint32)
        vecs = np.concatenate([base, start])
        want, words = D.inplace_delete(vecs, adj0, D.deleted_words(n + 1), sub, n, 1, O.L2, D.VISITED_AND_TOPK, NUM_TO_REPLACE, R,
                                       bench.ALPHA, K_VALUE, L_VALUE, batch_size=0)
        parity = {"ids": int(len(sub)), "rows_differing": int((got != want).any(1).sum()),
                  "table_equal": bool(np.array_equal(status, D.deleted_ids(words, n + 1)))}
        print(json.dumps({"parity": parity}), flush=True)
    out = {"card": name, "power_limit_and_max_sm_clock": power, "n": n, "nq": nq, "k": K, "L": L, "R": R,
           "num_to_replace": NUM_TO_REPLACE, "k_value": K_VALUE, "l_value": L_VALUE, "before": before, "settings": results,
           "parity": parity}
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    g.close()


if __name__ == "__main__":
    main()
