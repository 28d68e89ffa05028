"""MinMax compression behind a Hadamard transform against the Transform::Null path, on the device.

Two shapes: 1M x 128 behind PaddingHadamard (same, 4 bits) and 1M x 768 behind DoubleHadamard (same, 8 bits).  For each:
  * kernel times from torch.profiler (CUDA activity): hadamard_transform_kernel and minmax_compress_kernel, per call;
  * whole-call times from CUDA events around the host entry points (dab_minmax_compress on already transformed rows vs
    dab_minmax_compress_transformed), host copies included; median of --reps calls after one warm-up call;
  * the bytes the transform kernel must move (read input, write output) over its time.
The card's name and power limit are read in the same run and printed with the numbers.
usage: python tools/bench_minmax_transform.py [--n N] [--reps R] [--json PATH]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import diskann_b200 as dab


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def event_ms(fn, reps):
    fn()  # warm-up
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def kernel_ms(fn, reps):
    """mean device time per call of every kernel the calls launched, by kernel name"""
    fn()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ("kernel" in ev.key):
            out[ev.key] = ev.device_time_total / 1e3 / reps
    return out


def short(names):
    return {k.split("(")[0].split("::")[-1].split("<")[0]: v for k, v in names.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_minmax_transform: no CUDA device (no CPU fallback)")
    torch.cuda.init()
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}", flush=True)
    results = {"card": name, "power_limit_and_max_sm_clock": power, "n": args.n, "cases": []}
    rng = np.random.default_rng(0)
    for label, make, dim, nbits in (("PaddingHadamard same, 4-bit", dab.Transform.padding_hadamard, 128, 4),
                                    ("DoubleHadamard same, 8-bit", dab.Transform.double_hadamard, 768, 8)):
        t = make(dim, "same", 1)
        x = np.empty((args.n, dim), np.float32)
        for i in range(0, args.n, 1 << 17):
            x[i:i + (1 << 17)] = rng.standard_normal((min(1 << 17, args.n - i), dim), dtype=np.float32)
        tx = t.apply(x)
        rows_t, loss_t = dab.minmax_compress(x, nbits, 1.0, transform=t)
        rows_n, loss_n = dab.minmax_compress(tx, nbits, 1.0)
        same = bool(np.array_equal(rows_t, rows_n) and np.array_equal(loss_t.view(np.uint32), loss_n.view(np.uint32)))
        null_call = lambda: dab.minmax_compress(tx, nbits, 1.0)  # noqa: E731
        tr_call = lambda: dab.minmax_compress(x, nbits, 1.0, transform=t)  # noqa: E731
        e_null, e_tr = event_ms(null_call, args.reps), event_ms(tr_call, args.reps)
        k_null, k_tr = short(kernel_ms(null_call, args.reps)), short(kernel_ms(tr_call, args.reps))
        h_ms = k_tr.get("hadamard_transform_kernel", float("nan"))
        moved = args.n * (t.input_dim + t.output_dim) * 4
        case = {"case": label, "dim": dim, "nbits": nbits, "rows_equal_null_path_on_transformed_input": same,
                "call_ms_null": e_null, "call_ms_transformed": e_tr, "kernels_ms_null": k_null, "kernels_ms_transformed": k_tr,
                "transform_kernel_GB_per_s": moved / (h_ms * 1e-3) / 1e9}
        results["cases"].append(case)
        print(f"{label} {args.n} x {dim}: whole call {e_null:.1f} ms (Null) vs {e_tr:.1f} ms (transformed); "
              f"kernels Null {k_null}, transformed {k_tr}; transform kernel moves {case['transform_kernel_GB_per_s']:.0f} GB/s; "
              f"rows equal: {same}", flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
