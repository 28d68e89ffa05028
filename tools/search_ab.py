#!/usr/bin/env python3
"""A/B of the search benchmark between two built trees of this project, alternated in one process tree.

    python tools/search_ab.py BASE_TREE NEW_TREE [--runs 3] [--workload c2_1Mx128_f32_l2] [--steps 50] [--warmup 4]
                              [--dump-outputs] [--out results.jsonl]

Runs `bench.py --gpus 1` from BASE, NEW, BASE, NEW, ... (`--runs` times each; the CPU arm is skipped, it is not what
is compared), so that both trees see the same machine state in turn.  Every run records `ms_per_step` (batches in
flight), `config.serial.ms_per_step` (one batch at a time), recall and the parity gate, the GPU's name and power
limit (a read-only nvidia-smi query), and the occupancy of the search_kernel_v2 launches of its tree: launch grid,
registers per thread, dynamic shared memory and CTAs per SM, read from a torch.profiler trace of a small search at the
workload's shape (random graph; once per tree, since it depends on the compiled kernel and the layout, not on the run).
With --dump-outputs, what the last timed step returned is compared byte for byte across all runs of both trees.
Each tree must already be built (`__graft_entry__.build()`); nothing is written into either tree.
"""
import argparse
import glob
import json
import os
import statistics
import subprocess
import sys
import tempfile

PROBE = r"""
import json, os, sys, tempfile
import numpy as np
import torch
sys.path.insert(0, os.getcwd())
import bench
import diskann_b200 as dab

cfg = bench.WORKLOADS[sys.argv[1]]
dtype = {"f32": dab.DType.f32, "f16": dab.DType.f16, "i8": dab.DType.i8}[cfg["dtype"]]
metric = {"l2": dab.Metric.L2, "ip": dab.Metric.InnerProduct}[cfg["metric"]]
n, dim, md, nq = 50000, cfg["dim"], bench.max_degree(cfg["R"]), 10000
rng = np.random.default_rng(0)
vecs = rng.standard_normal((n + 1, dim), dtype=np.float32)
if cfg["dtype"] == "i8":
    vecs = np.clip(np.round(vecs * 25), -127, 127)
vecs = vecs.astype(bench.NP_DTYPE[cfg["dtype"]])
adj = np.empty((n + 1, md + 1), np.uint32)
adj[:, 0] = md
adj[:, 1:] = rng.integers(0, n + 1, (n + 1, md), dtype=np.uint32)
queries = vecs[rng.integers(0, n, nq)].copy()
launches = {}
with dab.GpuIndex(dtype, metric, dim, n, 1, md) as g:
    g.upload_vectors(vecs)
    g.upload_graph(adj)
    for mode in ("in_flight", "synchronous"):
        with tempfile.TemporaryDirectory() as tmp:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                if mode == "in_flight":
                    g.search_batch_async(0, queries, 10, cfg["l_search"])
                    g.wait(0)
                else:
                    g.search_batch(queries, 10, cfg["l_search"])
                torch.cuda.synchronize()
            prof.export_chrome_trace(os.path.join(tmp, "trace.json"))
            events = json.load(open(os.path.join(tmp, "trace.json")))["traceEvents"]
        for e in events:
            if e.get("cat") == "kernel" and "search_kernel" in e.get("name", ""):
                a = e.get("args", {})
                launches[mode] = {"kernel": e["name"], "grid": a.get("grid"), "block": a.get("block"),
                                  "registers_per_thread": a.get("registers per thread"),
                                  "dynamic_smem_bytes": a.get("shared memory"),
                                  "est_achieved_occupancy_pct": a.get("est. achieved occupancy %")}
                break
sms = torch.cuda.get_device_properties(0).multi_processor_count
for v in launches.values():
    if v["grid"] and "search_kernel_v2" in v["kernel"]:
        v["ctas_per_sm"] = v["grid"][0] / sms
print(json.dumps(launches))
"""


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = ([c.strip() for c in q.stdout.splitlines()[0].split(",")] + ["", "", ""])[:3] if q.stdout else ("", "", "")
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def child_env():
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    env.pop("PYTHONPATH", None)
    return env


def probe(tree, workload):
    r = subprocess.run([sys.executable, "-c", PROBE, workload], cwd=tree, capture_output=True, text=True, env=child_env())
    if r.returncode:
        raise SystemExit(f"occupancy probe failed in {tree}:\n{r.stderr[-3000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def bench_run(tree, args, dump_dir):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
           "--workload", args.workload, "--no-cpu-baseline"]
    if dump_dir:
        cmd += ["--dump-outputs", dump_dir]
    r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, env=child_env())
    if r.returncode:
        raise SystemExit(f"bench.py failed in {tree}:\n{r.stderr[-3000:]}")
    res = json.loads(r.stdout.strip().splitlines()[-1])
    conf = res["config"]
    return {"ms_per_step": res["ms_per_step"], "serial_ms_per_step": conf["serial"]["ms_per_step"],
            "recall_at_10": conf.get("recall_at_10"), "parity_gate": conf.get("parity_gate"), "clocks": res.get("clocks")}


def same_bytes(d0, d1):
    names = sorted(os.path.basename(p) for p in glob.glob(os.path.join(d0, "*.npy")))
    if not names or names != sorted(os.path.basename(p) for p in glob.glob(os.path.join(d1, "*.npy"))):
        return False
    return all(open(os.path.join(d0, f), "rb").read() == open(os.path.join(d1, f), "rb").read() for f in names)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("base")
    ap.add_argument("new")
    ap.add_argument("--runs", type=int, default=3, help="runs per tree, alternated")
    ap.add_argument("--workload", default="c2_1Mx128_f32_l2")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--dump-outputs", action="store_true", help="compare what both trees return, byte for byte")
    ap.add_argument("--out", default="", help="also append one JSON line per run (and the summary) to this file")
    args = ap.parse_args()
    trees = {"base": os.path.abspath(args.base), "new": os.path.abspath(args.new)}
    out = open(args.out, "a") if args.out else None

    def emit(obj):
        line = json.dumps(obj)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()

    occupancy = {k: probe(t, args.workload) for k, t in trees.items()}
    runs = {"base": [], "new": []}
    with tempfile.TemporaryDirectory(prefix="search_ab_") as tmp:
        for i in range(args.runs):
            for k in ("base", "new"):
                dump = os.path.join(tmp, f"{k}{i}") if args.dump_outputs else ""
                rec = dict(tree=k, run=i, workload=args.workload, gpu=gpu_info(), occupancy=occupancy[k],
                           **bench_run(trees[k], args, dump))
                runs[k].append(rec)
                emit(rec)
        identical = None
        if args.dump_outputs:
            dirs = [os.path.join(tmp, f"{k}{i}") for i in range(args.runs) for k in ("base", "new")]
            identical = all(same_bytes(dirs[0], d) for d in dirs[1:])

    ms = {k: [r["ms_per_step"] for r in v] for k, v in runs.items()}
    serial = {k: [r["serial_ms_per_step"] for r in v] for k, v in runs.items()}
    emit({"summary": args.workload,
          "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in ms.items()},
          "serial_ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in serial.items()},
          "new_over_base_median": statistics.median(ms["new"]) / statistics.median(ms["base"]),
          "serial_new_over_base_median": statistics.median(serial["new"]) / statistics.median(serial["base"]),
          "slowest_new_faster_than_fastest_base": max(ms["new"]) < min(ms["base"]),
          "outputs_byte_identical": identical})


if __name__ == "__main__":
    main()
