"""Graph search over the MinMax store against full precision and SQ-8, on the C2 workload of bench.py.

C2: 1M x 128 f32 rows, L2, a Vamana graph built on the device (R = 64, L_build = 100), batches of 10K queries.  Arms:
  * full precision: dab_search_batch_device;
  * SQ-8 traversal + full-precision rerank: dab_search_batch_sq_device;
  * MinMax 8-bit and 4-bit behind DoubleHadamard (TargetDim::Same, grid scale 1.0), rerank 0 and 1:
    dab_search_batch_minmax_device (the batch's queries are transformed and compressed inside the call);
each at several L.  Per (arm, L): ms per batch (CUDA events around one call on the index's stream, median of --reps after
two warm-up calls), QPS, recall@10 against the exact scan (dab_flat_knn), mean cmps and hops, and the bytes the traversal
reads per candidate (f32 row 512 + id; SQ-8 128; MinMax ceil(D * N / 8) + 16).  The card's name and power limit are read
in the same run and printed with the numbers.

--in-flight: one batch at a time against two batches in flight, at one L (--ls, first value): full precision, SQ-8 +
rerank and MinMax-8 (DoubleHadamard) + rerank on C2, and PQ-32 + rerank on small_200Kx128_i8_pq32.  Each mode rotates
--batches distinct query batches for --steps steps after --warmup steps: serially with the synchronous `_device` call on
the index's stream, in flight with the `_device_async` calls on slots 0 and 1 (a slot is joined with dab_wait just before
it takes its next batch).  CUDA events are recorded before the first step and after the last join; ms per batch is their
distance over the steps.  The outputs each slot holds after the last step must equal the synchronous call's on the same
batch, bit for bit.
usage: python tools/bench_minmax_search.py [--n N] [--nq NQ] [--ls 30,50,100,200] [--reps R] [--json PATH]
       python tools/bench_minmax_search.py --in-flight [--ls 100] [--steps 20] [--warmup 4] [--batches 4] [--json PATH]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import bench
import diskann_b200 as dab

K = 10


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def recall_at_k(gt, ids):
    return float(np.mean([len(np.intersect1d(gt[i, :K], ids[i, :K])) for i in range(gt.shape[0])]) / K)


def build_index(cfg, n, stream):
    """the workload's rows, start point (medoid copy) and device-built graph; PQ workloads also train and encode the table"""
    centers = bench.make_centers(cfg)
    base = bench.make_data(cfg, bench.SEED_BASE, n, centers)
    medoid = bench.find_medoid(base)
    dt, mt = {"f32": dab.DType.f32, "i8": dab.DType.i8}[cfg["dtype"]], {"l2": dab.Metric.L2, "ip": dab.Metric.InnerProduct}[cfg["metric"]]
    g = dab.GpuIndex(dt, mt, cfg["dim"], n, 1, bench.max_degree(cfg["R"]))
    g.set_stream(stream.cuda_stream)
    g.upload_vectors(base)
    g.upload_vectors(medoid[None, :], first=n)
    g.build(cfg["R"], cfg["l_build"], bench.ALPHA)
    if cfg["path"] == "pq":
        rng = np.random.default_rng(bench.SEED_PQ & 0xFFFFFFFF)
        sample = np.sort(rng.choice(n, size=min(cfg["pq_train"], n), replace=False))
        g.pq_train(base[sample].astype(np.float32), cfg["pq_chunks"], 256, 5, bench.SEED_PQ)
        g.pq_encode_all()
    return g, base, centers


def in_flight(args, name, power):
    """serial vs two batches in flight, per store (see the module docstring)"""
    L = int(args.ls.split(",")[0])
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    results = []

    def arm(label, g, cfg, nq, sync, launch):
        """sync(ptr, outs) / launch(slot, ptr, outs): the `_device` call and its `_device_async` twin"""
        centers = bench.make_centers(cfg)
        qs = [torch.from_numpy(bench.make_data(cfg, bench.SEED_QUERY + 97 * b, nq, centers)).cuda() for b in range(args.batches)]
        bufs = [[torch.empty((nq, K), dtype=torch.int32, device="cuda"), torch.empty((nq, K), dtype=torch.float32, device="cuda")]
                + [torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3)] for _ in range(3)]
        ptrs = [tuple(t.data_ptr() for t in b) for b in bufs]
        torch.cuda.synchronize()  # the slots' streams do not wait for torch's
        last = {}

        def serial(i):
            sync(qs[i % args.batches].data_ptr(), ptrs[0])

        def pipelined(i):
            s = i % 2
            g.wait(s)
            launch(s, qs[i % args.batches].data_ptr(), ptrs[s])
            last[s] = i % args.batches

        def timed(step, drain):
            for i in range(args.warmup):
                step(i)
            drain()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            a.synchronize()
            for i in range(args.warmup, args.warmup + args.steps):
                step(i)
            drain()
            b.record(stream)
            b.synchronize()
            return a.elapsed_time(b) / args.steps

        ms_serial = timed(serial, torch.cuda.synchronize)
        ms_flight = timed(pipelined, lambda: [g.wait(s) for s in (0, 1)])
        parity = True
        for s, bi in last.items():
            sync(qs[bi].data_ptr(), ptrs[2])
            torch.cuda.synchronize()
            parity &= all(torch.equal(x, y) for x, y in zip(bufs[s], bufs[2]))
        row = dict(arm=label, L=L, nq=nq, steps=args.steps, batches=args.batches, ms_per_batch_serial=round(ms_serial, 3),
                   ms_per_batch_in_flight=round(ms_flight, 3), speedup=round(ms_serial / ms_flight, 3), parity=bool(parity))
        results.append(row)
        print(json.dumps(row), flush=True)

    cfg = dict(bench.WORKLOADS["c2_1Mx128_f32_l2"])
    n, nq, dim = args.n or cfg["n"], args.nq or cfg["nq"], cfg["dim"]
    g, base, _ = build_index(cfg, n, stream)
    arm("full_precision", g, cfg, nq, lambda q, o: g.search_batch_device(q, nq, K, L, 1, *o),
        lambda s, q, o: g.search_batch_device_async(s, q, nq, K, L, 1, *o))
    mean, std = base.mean(0).astype(np.float32), float(base.std())
    shift = (mean - np.float32(2.5 * std)).astype(np.float32)
    g.upload_sq(8, shift, float(np.float32(5.0 * std)), float(np.dot(shift, shift)), 0.0)
    g.sq_encode_all()
    arm("sq8_rerank", g, cfg, nq, lambda q, o: g.search_batch_sq_device(q, nq, K, L, 1, *o, rerank=True),
        lambda s, q, o: g.search_batch_sq_device_async(s, q, nq, K, L, 1, *o, rerank=True))
    g.upload_minmax(8, 1.0, dab.Transform.double_hadamard(dim, "same", seed=7))
    g.minmax_encode_all()
    arm("minmax8_doublehadamard_rerank1", g, cfg, nq, lambda q, o: g.search_batch_minmax_device(q, nq, K, L, 1, *o, rerank=True),
        lambda s, q, o: g.search_batch_minmax_device_async(s, q, nq, K, L, 1, *o, rerank=True))
    g.close()
    cfg = dict(bench.WORKLOADS["small_200Kx128_i8_pq32"])
    g, _, _ = build_index(cfg, cfg["n"], stream)
    nq = cfg["nq"]
    arm("pq32_rerank (small_200Kx128_i8_pq32)", g, cfg, nq, lambda q, o: g.search_batch_pq_device(q, nq, K, L, 1, *o, rerank=True),
        lambda s, q, o: g.search_batch_pq_device_async(s, q, nq, K, L, 1, *o, rerank=True))
    g.close()
    summary = dict(gpu=name, power_limit_max_sm_clock=power, mode="in_flight", results=results)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    print(f"\n# {name}, power limit / max SM clock: {power}; L = {L}, k = 10, {args.steps} steps over {args.batches} batches")
    print(f"{'arm':40s} {'nq':>6s} {'serial ms':>10s} {'2 in flight':>12s} {'speedup':>8s} {'parity':>6s}")
    for r in results:
        print(f"{r['arm']:40s} {r['nq']:6d} {r['ms_per_batch_serial']:10.3f} {r['ms_per_batch_in_flight']:12.3f} {r['speedup']:8.3f} "
              f"{str(r['parity']):>6s}")
    if not all(r["parity"] for r in results):
        raise SystemExit("bench_minmax_search.py: a batch in flight differs from the synchronous call")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=0, help="point count (default: C2's 1M)")
    ap.add_argument("--nq", type=int, default=0, help="queries per batch (default: C2's 10K)")
    ap.add_argument("--ls", default="30,50,100,200")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default="")
    ap.add_argument("--in-flight", action="store_true", help="serial vs two batches in flight per store (module docstring)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--batches", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_minmax_search.py: no CUDA device")
    if args.in_flight:
        name, power = card()
        print(f"# {name}, power limit / max SM clock: {power}", flush=True)
        return in_flight(args, name, power)
    cfg = dict(bench.WORKLOADS["c2_1Mx128_f32_l2"])
    n = args.n or cfg["n"]
    nq = args.nq or cfg["nq"]
    dim = cfg["dim"]
    ls = [int(v) for v in args.ls.split(",")]
    name, power = card()
    print(f"# {name}, power limit / max SM clock: {power}", flush=True)

    centers = bench.make_centers(cfg)
    base = bench.make_data(cfg, bench.SEED_BASE, n, centers)
    medoid = bench.find_medoid(base)
    queries = bench.make_data(cfg, bench.SEED_QUERY, nq, centers)
    g = dab.GpuIndex(dab.DType.f32, dab.Metric.L2, dim, n, 1, bench.max_degree(cfg["R"]))
    stream = torch.cuda.Stream()  # the library and the events share one stream
    torch.cuda.set_stream(stream)
    g.set_stream(stream.cuda_stream)
    g.upload_vectors(base)
    g.upload_vectors(medoid[None, :], first=n)
    g.build(cfg["R"], cfg["l_build"], bench.ALPHA)
    gt, _ = g.flat_knn(queries, K)

    d_q = torch.from_numpy(queries).cuda()
    d_ids = torch.empty((nq, K), dtype=torch.int32, device="cuda")
    d_d = torch.empty((nq, K), dtype=torch.float32, device="cuda")
    d_c, d_cm, d_h = (torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(3))
    outs = (d_ids.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), d_cm.data_ptr(), d_h.data_ptr())

    def measure(arm, bytes_per_cand, call):
        for L in ls:
            call(L)
            call(L)
            times = []
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                call(L)
                b.record(stream)
                b.synchronize()
                times.append(a.elapsed_time(b))
            ms = float(np.median(times))
            ids = d_ids.cpu().numpy().view(np.uint32)
            row = dict(arm=arm, L=L, ms_per_batch=round(ms, 3), qps=round(nq / ms * 1e3), recall_at_10=round(recall_at_k(gt, ids), 4),
                       cmps_mean=round(float(d_cm.cpu().numpy().mean()), 1), hops_mean=round(float(d_h.cpu().numpy().mean()), 1),
                       bytes_per_candidate=bytes_per_cand, ms_spread=[round(min(times), 3), round(max(times), 3)])
            results.append(row)
            print(json.dumps(row), flush=True)

    results = []
    ptr = d_q.data_ptr()
    measure("full_precision", dim * 4 + 8, lambda L: g.search_batch_device(ptr, nq, K, L, 1, *outs))
    f32 = base
    mean, std = f32.mean(0).astype(np.float32), float(f32.std())
    shift = (mean - np.float32(2.5 * std)).astype(np.float32)
    g.upload_sq(8, shift, float(np.float32(5.0 * std)), float(np.dot(shift, shift)), 0.0)
    g.sq_encode_all()
    measure("sq8_rerank", dim, lambda L: g.search_batch_sq_device(ptr, nq, K, L, 1, *outs, rerank=True))
    t = dab.Transform.double_hadamard(dim, "same", seed=7)
    for nbits in (8, 4):
        g.upload_minmax(nbits, 1.0, t)
        g.minmax_encode_all()
        for rerank in (False, True):
            measure(f"minmax{nbits}_doublehadamard_rerank{int(rerank)}", (dim * nbits + 7) // 8 + 16,
                    lambda L: g.search_batch_minmax_device(ptr, nq, K, L, 1, *outs, rerank=rerank))
    g.close()
    summary = dict(gpu=name, power_limit_max_sm_clock=power, n=n, nq=nq, dim=dim, results=results)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    print(f"\n# {name}, power limit / max SM clock: {power}; n = {n}, {nq} queries per batch, k = 10")
    print(f"{'arm':40s} {'L':>5s} {'ms/batch':>9s} {'QPS':>10s} {'recall@10':>9s} {'cmps':>7s} {'B/cand':>6s}")
    for r in results:
        print(f"{r['arm']:40s} {r['L']:5d} {r['ms_per_batch']:9.3f} {r['qps']:10d} {r['recall_at_10']:9.4f} {r['cmps_mean']:7.1f} "
              f"{r['bytes_per_candidate']:6d}")


if __name__ == "__main__":
    main()
